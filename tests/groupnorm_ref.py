"""fp64 restatement of the joint-frame GroupNorm path (model/xunet.py:46-61, 82-84) stage by stage, as the CUDA kernels split it.

Tensors are channels-last (N, H, W, C) with N = 2B: frames 2b and 2b+1 are one sample, and GroupNorm(32) pools each group over
both frames.  The stages and what each kernel stores:
  cstats        per-(sample, channel) [sum y, sum y^2] of a producer's stored output          (conv EPI 1, attention, gn_cstats)
  table         per-(sample, channel) {rstd, -mean*rstd, gamma, beta}                          (gn_apply params_out)
  forward       y = act(yhat), yhat = xhat*gamma + beta, xhat = (x - mean)*rstd, then RS_DOWN / RS_UP   (gn_apply)
  dyhat         the gradient w.r.t. yhat from the gradient of the activation, and the FiLM gradient de   (conv EPI 2 / 3)
  bcs           per-(sample, channel) [sum dyhat*xhat, sum dyhat]                              (conv EPI 2 / 3, gn_bwd_reduce)
  dx            rstd*(gamma*dyhat - S1/cnt - xhat*S2/cnt), S1 = sum_group gamma*sum dyhat, S2 = sum_group gamma*sum dyhat*xhat
  dgamma, dbeta the channel sums over all samples
"""
import torch

GROUPS = 32
EPS = 1e-6            # XU_GN_EPS
PLAIN, SWISH, FILM = 0, 1, 2
RS_NONE, RS_DOWN, RS_UP = 0, 1, 2


def _split(t):
    """(N, H, W, C) -> (B, 2HW, C): one row per sample, both frames."""
    N, H, W, C = t.shape
    return t.reshape(N // 2, 2 * H * W, C)


def _per_channel(stat, N, H, W):
    """(B, C) -> broadcastable against (N, H, W, C): sample b's value on frames 2b and 2b+1."""
    return stat.repeat_interleave(2, dim=0)[:, None, None, :]


def group_of(C):
    return torch.arange(C) // (C // GROUPS)


def cstats(y):
    """(N, H, W, C) -> (B, C, 2) [sum y, sum y^2] over both frames of each sample."""
    t = _split(y.double())
    return torch.stack([t.sum(1), (t * t).sum(1)], dim=-1)


def group_sums(cs):
    """(B, C, 2) channel sums -> (B, 32, 2) group sums."""
    B, C, _ = cs.shape
    return cs.reshape(B, GROUPS, C // GROUPS, 2).sum(2)


def count(H, W, C):
    """elements per group and sample: both frames, C/32 channels"""
    return 2 * H * W * (C // GROUPS)


def mean_rstd_from_sums(gs, H, W, C):
    """(B, 32, 2) group sums -> per-(sample, channel) mean and rstd (B, C), with the kernels' E[x^2] - mean^2 variance."""
    cnt = count(H, W, C)
    mean = gs[..., 0] / cnt
    var = torch.clamp(gs[..., 1] / cnt - mean * mean, min=0.)
    rstd = 1. / torch.sqrt(var + EPS)
    g = group_of(C)
    return mean[:, g], rstd[:, g]


def mean_rstd(x):
    """Exact two-pass statistics of x (N, H, W, C): per-(sample, channel) mean and rstd (B, C)."""
    N, H, W, C = x.shape
    t = x.double().reshape(N // 2, 2 * H * W, GROUPS, C // GROUPS)
    mean = t.mean(dim=(1, 3))
    var = ((t - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    g = group_of(C)
    return mean[:, g], (1. / torch.sqrt(var + EPS))[:, g]


def table(mean, rstd, gamma, beta):
    """(B, C, 4) {rstd, -mean*rstd, gamma, beta}: xhat = x*rstd + (-mean*rstd), yhat = xhat*gamma + beta."""
    B, C = mean.shape
    return torch.stack([rstd, -mean * rstd, gamma.double().expand(B, C), beta.double().expand(B, C)], dim=-1)


def xhat(x, mean, rstd):
    N, H, W, C = x.shape
    return (x.double() - _per_channel(mean, N, H, W)) * _per_channel(rstd, N, H, W)


def swish(u):
    return u * torch.sigmoid(u)


def swish_grad(u):
    s = torch.sigmoid(u)
    return s * (1. + u * (1. - s))


def keep_scale(drop_rate):
    return 1. / (1. - float(torch.tensor(drop_rate, dtype=torch.float32)))


def resample(a, rs):
    """RS_DOWN: 2x2 mean (after the activation); RS_UP: nearest 2x."""
    if rs == RS_DOWN:
        N, H, W, C = a.shape
        return a.reshape(N, H // 2, 2, W // 2, 2, C).mean(dim=(2, 4))
    if rs == RS_UP:
        return a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return a


def resample_adjoint(g, rs):
    """gradient w.r.t. the activation (before resampling) from the gradient of the resampled output"""
    if rs == RS_DOWN:
        return 0.25 * g.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    if rs == RS_UP:
        N, H2, W2, C = g.shape
        return g.reshape(N, H2 // 2, 2, W2 // 2, 2, C).sum(dim=(2, 4))
    return g


def forward(x, gamma, beta, mode, rs=RS_NONE, e=None, keep=None, drop_rate=0., mean=None, rstd=None):
    """The GroupNorm output.  e (N, H, W, 2C) = [scale | shift] (FILM); keep: 0/1 dropout mask of (N, H, W, C) or None.
    mean / rstd (B, C): the statistics to use (default: the exact ones of x)."""
    if mean is None:
        mean, rstd = mean_rstd(x)
    yh = xhat(x, mean, rstd) * gamma.double() + beta.double()
    if mode == PLAIN:
        a = yh
    elif mode == SWISH:
        a = swish(yh)
    else:
        C = x.shape[-1]
        sc, sh = e.double()[..., :C], e.double()[..., C:]
        a = swish(yh * (1. + sc) + sh)
        if keep is not None:
            a = a * keep.double() * keep_scale(drop_rate)
    return resample(a, rs)


def dyhat(g_act, x, gamma, beta, mode, e=None, keep=None, drop_rate=0., mean=None, rstd=None):
    """(dyhat, de) from g_act, the gradient w.r.t. the activation at input resolution (resample_adjoint of the output's).
    de (N, H, W, 2C) = [du * yhat | du] for FILM (du: gradient w.r.t. the swish input), else None."""
    if mean is None:
        mean, rstd = mean_rstd(x)
    yh = xhat(x, mean, rstd) * gamma.double() + beta.double()
    g = g_act.double()
    if mode == PLAIN:
        return g, None
    if mode == SWISH:
        return g * swish_grad(yh), None
    C = x.shape[-1]
    sc, sh = e.double()[..., :C], e.double()[..., C:]
    if keep is not None:
        g = g * keep.double() * keep_scale(drop_rate)
    du = g * swish_grad(yh * (1. + sc) + sh)
    return du * (1. + sc), torch.cat([du * yh, du], dim=-1)


def bcs(dyh, xh):
    """(B, C, 2) [sum dyhat*xhat, sum dyhat] over both frames of each sample."""
    a, b = _split(dyh.double()), _split(xh.double())
    return torch.stack([(a * b).sum(1), a.sum(1)], dim=-1)


def dx(dyh, xh, rstd, gamma, sums):
    """rstd*(gamma*dyhat - S1/cnt - xhat*S2/cnt) with S1 = sum_group gamma*sum dyhat, S2 = sum_group gamma*sum dyhat*xhat.
    Also returns the three terms' magnitude rstd*(|gamma dyhat| + |S1/cnt| + |xhat S2/cnt|), the scale of its cancellation."""
    N, H, W, C = dyh.shape
    cnt = count(H, W, C)
    gm = gamma.double()
    B = N // 2
    s1 = (gm * sums[..., 1]).reshape(B, GROUPS, -1).sum(-1)[:, group_of(C)] / cnt
    s2 = (gm * sums[..., 0]).reshape(B, GROUPS, -1).sum(-1)[:, group_of(C)] / cnt
    r, s1, s2 = (_per_channel(t, N, H, W) for t in (rstd, s1, s2))
    t1, t3 = gm * dyh.double(), xh.double() * s2
    return r * (t1 - s1 - t3), r * (t1.abs() + s1.abs() + t3.abs())


def group_bsums(gamma, sums):
    """(B, 32, 2) [S1, S2] = [sum_group gamma*sum dyhat, sum_group gamma*sum dyhat*xhat]: what gn_bwd_reduce stores to bstats"""
    B, C, _ = sums.shape
    gm = gamma.double()
    return torch.stack([(gm * sums[..., 1]).reshape(B, GROUPS, -1).sum(-1), (gm * sums[..., 0]).reshape(B, GROUPS, -1).sum(-1)],
                       dim=-1)


def dgamma_dbeta(sums):
    return sums[..., 0].sum(0), sums[..., 1].sum(0)
