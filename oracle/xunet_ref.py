"""CPU ORACLE for the X-UNet hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

    PARITY UNPINNED: the reference (JAX/Flax) cannot be imported in the
    project's environment (jax, flax, optax, visu3d are absent and there is no network) and the reference
    ships no tests / golden vectors.  This file is a line-by-line CPU restatement of
    `model/xunet.py`, `train.py:36-76` and `sampling.py:16-53,73-76,119-151` in torch-CPU
    (fp64 = truth, fp32 = what JAX-CPU would produce and the timed CPU baseline).  Its
    pins are the known-answer / metamorphic properties derivable from the reference source
    (tests/test_oracle.py) and the fp64 golden vectors under tests/golden/.

    Round 2 additions: (i) every primitive below is cross-checked on CPU against an INDEPENDENT
    implementation (torch.nn.functional.group_norm / scaled_dot_product_attention / avg_pool2d /
    interpolate / conv2d with explicit padding, tests/test_oracle.py::test_primitive_*), so the
    oracle is no longer "one author's reading, twice"; (ii) `Bf16Emulation` restates WHERE the
    CUDA engine rounds to bf16 (stored activations / gradients, tensor-core weight shadows,
    attention probabilities) so the product dtype can be held to a tight tolerance too.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / --impl reference
legs may import this module.  Nothing under `novel_view_synthesis_3d_b200/` imports it.

Third-party semantics restated here (see SURVEY.md 8(c)):
  flax 0.6.4   nn.Conv ('SAME', XLA padding rule), nn.Dense, nn.DenseGeneral, nn.GroupNorm
               (eps 1e-6, biased var = max(0, E[x^2]-E[x]^2)), nn.dot_product_attention,
               nn.avg_pool (VALID), nn.Dropout, nn.swish, lecun_normal.
  optax        adam (b1 .9, b2 .999, eps 1e-8, eps_root 0).
  visu3d 1.3.0 Camera.rays(): pos = t, dir = normalize(R K^-1 [px, 1]) at pixel centres.

Layout conventions (identical to Flax): activations (B, F=2, H, W, C); conv kernel
(1, 3, 3, I, O); Dense kernel (I, O); DenseGeneral kernel (C, heads, head_dim).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from dataclasses import dataclass
from typing import Callable, Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

SQRT2 = math.sqrt(2.0)
POSE_EMB_DIM = 144  # 3 + 6*15 (pos)  +  3 + 6*8 (dir)   model/xunet.py:162-164


# --------------------------------------------------------------------------------------
# config  (model/xunet.py:205-215; ch_mult / attn_resolutions are class attributes there)
# --------------------------------------------------------------------------------------
@dataclass(frozen=True)
class RefConfig:
    ch: int = 32
    ch_mult: Tuple[int, ...] = (1, 2)
    emb_ch: int = 32
    num_res_blocks: int = 2
    attn_resolutions: Tuple[int, ...] = (8, 16, 32)
    attn_heads: int = 4
    dropout: float = 0.1
    use_pos_emb: bool = False
    use_ref_pose_emb: bool = False


SMALL = RefConfig()
FULL = RefConfig(ch=256, ch_mult=(1, 2, 2, 4), emb_ch=1024, num_res_blocks=3,
                 attn_resolutions=(8, 16, 32), attn_heads=8)


# --------------------------------------------------------------------------------------
# bf16 emulation policy (test infrastructure for the product dtype; identity when absent)
# --------------------------------------------------------------------------------------
def _bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _Store(torch.autograd.Function):
    """A tensor the engine keeps in HBM as bf16: value rounded in forward, its gradient rounded in backward."""
    @staticmethod
    def forward(ctx, x):
        return _bf16(x)

    @staticmethod
    def backward(ctx, g):
        return _bf16(g)


class _RoundSTE(torch.autograd.Function):
    """Rounded operand of a tensor-core MMA whose gradient is NOT stored rounded (weight shadows, attention P)."""
    @staticmethod
    def forward(ctx, x):
        return _bf16(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _GradRound(torch.autograd.Function):
    """Identity whose incoming gradient is rounded (dS before the dQ / dK MMAs)."""
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return _bf16(g)


class Bf16Emulation:
    """Where libxunet_b200's bf16 mode rounds (DESIGN.md section 3 'Precision'): every activation tensor and activation
    gradient is stored as bf16 (`store`); conv / dense / q|k|v kernels reach the tensor cores as bf16 shadows of the fp32
    masters (`weight`; the two 3-channel direct convolutions and all biases / GroupNorm affine / log-SNR MLP stay fp32);
    attention probabilities are rounded for the PV and dV products while the row sum uses the unrounded values (`prob`);
    dS is rounded before the dQ / dK products (`grad_only`).  Accumulation, statistics, softmax state, loss: fp32 in the
    engine, the oracle's compute dtype here."""
    store = staticmethod(_Store.apply)
    weight = staticmethod(_RoundSTE.apply)
    prob = staticmethod(_RoundSTE.apply)
    grad_only = staticmethod(_GradRound.apply)


class _NoEmulation:
    store = weight = prob = grad_only = staticmethod(lambda x: x)


_EXACT = _NoEmulation()


# --------------------------------------------------------------------------------------
# small ops
# --------------------------------------------------------------------------------------
def swish(x):  # nn.swish, model/xunet.py:9
    return x * torch.sigmoid(x)


def nearest_neighbor_upsample(h):  # model/xunet.py:14-18
    B, Fr, H, W, C = h.shape
    h = h.reshape(B, Fr, H, 1, W, 1, C).expand(B, Fr, H, 2, W, 2, C)
    return h.reshape(B, Fr, H * 2, W * 2, C)


def avgpool_downsample(h, k=2):  # model/xunet.py:20-21 (nn.avg_pool window (1,k,k), VALID)
    B, Fr, H, W, C = h.shape
    h = h[:, :, :H // k * k, :W // k * k]
    h = h.reshape(B, Fr, H // k, k, W // k, k, C)
    return h.mean(dim=(3, 5))


def posenc_ddpm(timesteps, emb_ch: int, max_time=1000.):  # model/xunet.py:23-35
    dtype = timesteps.dtype
    timesteps = timesteps * (1000. / max_time)
    half_dim = emb_ch // 2
    emb = np.log(10000) / (half_dim - 1)
    emb = torch.exp(torch.arange(half_dim, dtype=dtype) * -emb)
    emb = timesteps[..., None] * emb
    return torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)


def posenc_nerf(x, min_deg=0, max_deg=15):  # model/xunet.py:37-44
    """The reference computes the ARGUMENT of sin in fp32 (JAX x64 off): x is fp32, x*2^i is exact, and `xb + pi/2`
    is an fp32 add whose rounding (ulp 2e-3 at |xb|~2e4) is part of the function being matched.  The argument is
    therefore always formed in fp32 here; only sin() itself runs in the oracle's compute dtype."""
    if min_deg == max_deg:
        return x
    dtype = x.dtype
    x32 = x.to(torch.float32)
    scales = torch.tensor([2.0 ** i for i in range(min_deg, max_deg)], dtype=torch.float32)
    # x[..., None, :] * scales[:, None] -> (..., n_scales, 3) -> (..., 3 n): scale-major
    xb = (x32[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
    half_pi = torch.tensor(np.pi / 2., dtype=torch.float32)
    arg = torch.cat([xb, xb + half_pi], dim=-1)
    emb = torch.sin(arg.to(dtype))
    return torch.cat([x32.to(dtype), emb], dim=-1)


def camera_rays(R, t, K, H, W, convention='v3d130_ij'):
    """visu3d 1.3.0  Camera(spec=PinholeCamera(resolution=(H,W), K), world_from_cam=Transform(R,t)).rays()
    (model/xunet.py:159-161).  pos = t broadcast; dir = normalize(R @ K^-1 @ [p0, p1, 1]).

    convention 'v3d130_ij': pixel coordinate fed to K^-1 is (i+.5, j+.5) = (row, col)   [visu3d <= 1.3]
    convention 'opencv_uv': pixel coordinate is (u, v) = (col+.5, row+.5)               [visu3d >= 1.4]
    Returns pos, dir of shape (B, H, W, 3).
    """
    B = R.shape[0]
    dtype = R.dtype
    ii, jj = torch.meshgrid(torch.arange(H, dtype=dtype) + 0.5,
                            torch.arange(W, dtype=dtype) + 0.5, indexing='ij')
    if convention == 'v3d130_ij':
        p0, p1 = ii, jj
    elif convention == 'opencv_uv':
        p0, p1 = jj, ii
    else:
        raise ValueError(convention)
    px = torch.stack([p0, p1, torch.ones_like(p0)], dim=-1)            # (H, W, 3)
    Kinv = torch.linalg.inv(K.double()).to(dtype)                      # (B, 3, 3)
    cam = torch.einsum('bij,hwj->bhwi', Kinv, px)
    world = torch.einsum('bij,bhwj->bhwi', R, cam)
    world = world / torch.linalg.norm(world, dim=-1, keepdim=True)
    pos = t[:, None, None, :].expand(B, H, W, 3)
    return pos, world


def same_pad(in_size: int, k: int, s: int) -> Tuple[int, int]:
    """XLA 'SAME' padding rule used by flax nn.Conv."""
    out = -(-in_size // s)
    total = max((out - 1) * s + k - in_size, 0)
    lo = total // 2
    return lo, total - lo


def conv_1x3x3(h, kernel, bias, stride=1):
    """nn.Conv(features, kernel_size=(1,3,3), strides=(1,s,s)) on (B,F,H,W,C); kernel (1,3,3,I,O)."""
    B, Fr, H, W, C = h.shape
    x = h.reshape(B * Fr, H, W, C).permute(0, 3, 1, 2)
    w = kernel[0].permute(3, 2, 0, 1)                                  # (O, I, 3, 3)
    pl_h, ph_h = same_pad(H, 3, stride)
    pl_w, ph_w = same_pad(W, 3, stride)
    x = F.pad(x, (pl_w, ph_w, pl_h, ph_h))
    y = F.conv2d(x, w, bias, stride=stride)
    y = y.permute(0, 2, 3, 1)
    return y.reshape(B, Fr, y.shape[1], y.shape[2], y.shape[3])


def dense(x, p):  # nn.Dense: kernel (I, O)
    return x @ p['kernel'] + p['bias']


def group_norm(h, p, eps=1e-6, num_groups=32):
    """model/xunet.py:46-52 -> nn.GroupNorm(num_groups=32) on (B,2,H,W,C): stats over (F,H,W,C/32) jointly."""
    p = p['GroupNorm_0']
    B, Fr, H, W, C = h.shape
    assert C % num_groups == 0
    x = h.reshape(B, Fr * H * W, num_groups, C // num_groups)
    mean = x.mean(dim=(1, 3), keepdim=True)
    mean2 = (x * x).mean(dim=(1, 3), keepdim=True)
    var = torch.clamp(mean2 - mean * mean, min=0.)
    y = (x - mean) * torch.rsqrt(var + eps)
    y = y.reshape(B, Fr, H, W, C)
    return y * p['scale'] + p['bias']


def film(h, emb, p, emu=_EXACT):  # model/xunet.py:54-61
    # engine: swish(emb) is one stored tensor per level; the Dense output (scale | shift) is stored too
    e = emu.store(dense(emu.store(swish(emb)), {'kernel': emu.weight(p['Dense_0']['kernel']), 'bias': p['Dense_0']['bias']}))
    scale, shift = torch.chunk(e, 2, dim=-1)
    return h * (1. + scale) + shift


def resnet_block(h_in, emb, p, *, features=None, resample=None, dropout=0., train=False,
                 drop_mask=None, emu=_EXACT):
    """model/xunet.py:63-92.  drop_mask: keep-mask (bool/0-1) of the Dropout input's shape, or None.
    emu: rounding points of the bf16 engine (GN+swish(+resample) output, Conv_0 output, FiLM+swish+dropout output, the
    1x1 skip projection, and the block output after the residual combine)."""
    C = h_in.shape[-1]
    features = C if features is None else features
    h = swish(group_norm(h_in, p['GroupNorm_0']))
    if resample is not None:
        updown = {'up': nearest_neighbor_upsample, 'down': avgpool_downsample}[resample]
        h = updown(h)
        h_in = emu.store(updown(h_in))
    h = emu.store(h)
    h = emu.store(conv_1x3x3(h, emu.weight(p['Conv_0']['kernel']), p['Conv_0']['bias']))
    h = film(group_norm(h, p['GroupNorm_1']), emb, p['FiLM_0'], emu)
    h = swish(h)
    if train and dropout > 0.:
        assert drop_mask is not None, 'oracle needs an explicit dropout keep-mask when train=True'
        h = torch.where(drop_mask.bool(), h / (1. - dropout), torch.zeros_like(h))
    h = emu.store(h)
    h = conv_1x3x3(h, emu.weight(p['Conv_1']['kernel']), p['Conv_1']['bias'])
    if C != features:
        h_in = emu.store(dense(h_in, {'kernel': emu.weight(p['Dense_0']['kernel']), 'bias': p['Dense_0']['bias']}))
    return emu.store((h + h_in) / SQRT2)


def attn_layer(q_in, kv_in, p, heads, emu=_EXACT):  # model/xunet.py:94-103
    def proj(x, pp):  # DenseGeneral((heads, hd)): kernel (C, heads, hd), bias (heads, hd)
        return emu.store(torch.einsum('blc,chd->blhd', x, emu.weight(pp['kernel'])) + pp['bias'])
    q = proj(q_in, p['DenseGeneral_0'])
    k = proj(kv_in, p['DenseGeneral_1'])
    v = proj(kv_in, p['DenseGeneral_2'])
    hd = q.shape[-1]
    q = q / math.sqrt(hd)
    w = emu.grad_only(torch.einsum('bqhd,bkhd->bhqk', q, k))
    w = emu.prob(torch.softmax(w, dim=-1))
    return torch.einsum('bhqk,bkhd->bqhd', w, v)


def attn_block(h_in, p, attn_type, heads, emu=_EXACT):  # model/xunet.py:105-127
    B, Fr, H, W, C = h_in.shape
    h = emu.store(group_norm(h_in, p['GroupNorm_0']))
    h0 = h[:, 0].reshape(B, H * W, C)
    h1 = h[:, 1].reshape(B, H * W, C)
    pl = p['AttnLayer_0']
    if attn_type == 'self':
        o0 = attn_layer(h0, h0, pl, heads, emu)
        o1 = attn_layer(h1, h1, pl, heads, emu)
    elif attn_type == 'cross':
        o0 = attn_layer(h0, h1, pl, heads, emu)
        o1 = attn_layer(h1, h0, pl, heads, emu)
    else:
        raise NotImplementedError(attn_type)
    h = torch.stack([o0, o1], dim=1).reshape(B, Fr, H, W, -1)
    return emu.store((h + h_in) / SQRT2)


def xunet_block(x, emb, p, *, features, use_attn, heads, dropout, train, drop_mask, emu=_EXACT):  # :129-140
    h = resnet_block(x, emb, p['ResnetBlock_0'], features=features, dropout=dropout, train=train,
                     drop_mask=drop_mask, emu=emu)
    if use_attn:
        h = attn_block(h, p['AttnBlock_0'], 'self', heads, emu)
        h = attn_block(h, p['AttnBlock_1'], 'cross', heads, emu)
    return h


def conditioning(p, batch, cond_mask, cfg: RefConfig, *, rays=None, ray_convention='v3d130_ij', emu=_EXACT):
    """ConditioningProcessor.__call__  model/xunet.py:150-203.

    rays: optional ((pos1, dir1), (pos2, dir2)) each (B,H,W,3) to bypass the visu3d restatement."""
    x = batch['x']
    B, H, W, C = x.shape
    dtype = x.dtype
    logsnr = torch.clamp(batch['logsnr'].to(dtype), -20., 20.)
    logsnr = 2. * torch.atan(torch.exp(-logsnr / 2.)) / np.pi
    logsnr_emb = posenc_ddpm(logsnr, emb_ch=cfg.emb_ch, max_time=1.)
    logsnr_emb = dense(logsnr_emb, p['Dense_0'])
    logsnr_emb = dense(swish(logsnr_emb), p['Dense_1'])
    if rays is None:
        rays = (camera_rays(batch['R1'].to(dtype), batch['t1'].to(dtype), batch['K'].to(dtype), H, W, ray_convention),
                camera_rays(batch['R2'].to(dtype), batch['t2'].to(dtype), batch['K'].to(dtype), H, W, ray_convention))
    embs = []
    for pos, d in rays:
        embs.append(torch.cat([posenc_nerf(pos.to(dtype), 0, 15), posenc_nerf(d.to(dtype), 0, 8)], dim=-1))
    pose_emb = torch.stack(embs, dim=1)                                # (B, 2, H, W, 144)
    D = pose_emb.shape[-1]
    assert D == POSE_EMB_DIM
    assert cond_mask.shape == (B,)
    cm = cond_mask.reshape(B, 1, 1, 1, 1).to(torch.bool)
    pose_emb = torch.where(cm, pose_emb, torch.zeros_like(pose_emb))
    if cfg.use_pos_emb:
        pose_emb = pose_emb + p['pos_emb'][None, None]
    if cfg.use_ref_pose_emb:
        first = p['ref_pose_emb_first'][None, None, None, None]
        other = p['ref_pose_emb_other'][None, None, None, None]
        pose_emb = pose_emb + torch.cat([first, other], dim=1)
    pose_emb = emu.store(pose_emb)
    pose_embs = []
    for i_level in range(len(cfg.ch_mult)):
        pc = p[f'Conv_{i_level}']
        pose_embs.append(emu.store(conv_1x3x3(pose_emb, emu.weight(pc['kernel']), pc['bias'], stride=2 ** i_level)))
    return logsnr_emb, pose_embs


def xunet_forward(params, batch, cond_mask, cfg: RefConfig = SMALL, *, train=False,
                  drop_mask_fn: Optional[Callable] = None, rays=None, ray_convention='v3d130_ij',
                  both_frames=False, taps: Optional[dict] = None, emu=None):
    """XUNet.__call__  model/xunet.py:218-280.  Returns eps_hat (B,H,W,3) for the target frame
    (or both frames (B,2,H,W,3) if both_frames).  drop_mask_fn(resblock_index, shape)->keep mask.
    `taps`, if a dict, receives named intermediate activations.  emu: None (exact) or Bf16Emulation()."""
    emu = emu or _EXACT
    x = batch['x']
    dtype = x.dtype
    B, H, W, C = x.shape
    L = len(cfg.ch_mult)
    logsnr_emb, pose_embs = conditioning(params['ConditioningProcessor_0'], batch, cond_mask, cfg,
                                         rays=rays, ray_convention=ray_convention, emu=emu)
    if taps is not None:
        taps['logsnr_emb'] = logsnr_emb
        for i, pe in enumerate(pose_embs):
            taps[f'pose_emb_{i}'] = pe
    lemb = logsnr_emb[:, None, None, None, :]

    counters = {'xb': 0, 'rb': 0, 'res': 0}

    def mask_for(shape):
        idx = counters['res']
        counters['res'] += 1
        if train and cfg.dropout > 0.:
            return drop_mask_fn(idx, shape)
        return None

    def xblock(h, emb, features, use_attn):
        name = f"XUNetBlock_{counters['xb']}"
        counters['xb'] += 1
        Bh, Fh, Hh, Wh, _ = h.shape
        m = mask_for((Bh, Fh, Hh, Wh, features))
        out = xunet_block(h, emb, params[name], features=features, use_attn=use_attn, heads=cfg.attn_heads,
                          dropout=cfg.dropout, train=train, drop_mask=m, emu=emu)
        if taps is not None:
            taps[name] = out
        return out

    def rblock(h, emb, resample):
        name = f"ResnetBlock_{counters['rb']}"
        counters['rb'] += 1
        Bh, Fh, Hh, Wh, Ch = h.shape
        Ho = Hh * 2 if resample == 'up' else Hh // 2
        Wo = Wh * 2 if resample == 'up' else Wh // 2
        m = mask_for((Bh, Fh, Ho, Wo, Ch))
        out = resnet_block(h, emb, params[name], resample=resample, dropout=cfg.dropout, train=train, drop_mask=m, emu=emu)
        if taps is not None:
            taps[name] = out
        return out

    h = emu.store(torch.stack([batch['x'].to(dtype), batch['z'].to(dtype)], dim=1))
    h = emu.store(conv_1x3x3(h, params['Conv_0']['kernel'], params['Conv_0']['bias']))      # direct 3-channel kernel: fp32 weights
    hs = [h]
    for i_level in range(L):
        emb = lemb + pose_embs[i_level]
        for _ in range(cfg.num_res_blocks):
            use_attn = h.shape[2] in cfg.attn_resolutions
            h = xblock(h, emb, cfg.ch * cfg.ch_mult[i_level], use_attn)
            hs.append(h)
        if i_level != L - 1:
            emb = lemb + pose_embs[i_level + 1]
            h = rblock(h, emb, 'down')
            hs.append(h)
    # middle (features uses the leaked loop variable i_level == L-1, model/xunet.py:252)
    emb = lemb + pose_embs[-1]
    use_attn = h.shape[2] in cfg.attn_resolutions
    h = xblock(h, emb, cfg.ch * cfg.ch_mult[L - 1], use_attn)
    for i_level in reversed(range(L)):
        emb = lemb + pose_embs[i_level]
        for _ in range(cfg.num_res_blocks + 1):
            use_attn = hs[-1].shape[2] in cfg.attn_resolutions
            h = torch.cat([h, hs.pop()], dim=-1)
            h = xblock(h, emb, cfg.ch * cfg.ch_mult[i_level], use_attn)
        if i_level != 0:
            emb = lemb + pose_embs[i_level - 1]
            h = rblock(h, emb, 'up')
    assert not hs
    h = emu.store(swish(group_norm(h, params['GroupNorm_0'])))
    out = emu.store(conv_1x3x3(h, params['Conv_1']['kernel'], params['Conv_1']['bias']))      # direct 3-channel kernel
    return out if both_frames else out[:, 1]


# --------------------------------------------------------------------------------------
# parameter tree (Flax auto-naming; SURVEY.md Appendix A) and init (train.py:36-47)
# --------------------------------------------------------------------------------------
def param_shapes(cfg: RefConfig, S: int) -> "OrderedDict[str, Tuple[int, ...]]":
    """Flat 'a/b/c' -> shape map in module creation order, derived by walking model/xunet.py:218-280."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    E, D, L = cfg.emb_ch, POSE_EMB_DIM, len(cfg.ch_mult)

    def add(name, shape):
        assert name not in out, name
        out[name] = tuple(shape)

    def conv(prefix, cin, cout):
        add(prefix + '/kernel', (1, 3, 3, cin, cout))
        add(prefix + '/bias', (cout,))

    def dense_(prefix, cin, cout):
        add(prefix + '/kernel', (cin, cout))
        add(prefix + '/bias', (cout,))

    def gn(prefix, c):
        add(prefix + '/GroupNorm_0/scale', (c,))
        add(prefix + '/GroupNorm_0/bias', (c,))

    def resblock(prefix, cin, feat):
        gn(prefix + '/GroupNorm_0', cin)
        conv(prefix + '/Conv_0', cin, feat)
        gn(prefix + '/GroupNorm_1', feat)
        dense_(prefix + '/FiLM_0/Dense_0', E, 2 * feat)
        conv(prefix + '/Conv_1', feat, feat)
        if cin != feat:
            dense_(prefix + '/Dense_0', cin, feat)

    def attnblock(prefix, c):
        gn(prefix + '/GroupNorm_0', c)
        hd = c // cfg.attn_heads
        for i in range(3):
            add(prefix + f'/AttnLayer_0/DenseGeneral_{i}/kernel', (c, cfg.attn_heads, hd))
            add(prefix + f'/AttnLayer_0/DenseGeneral_{i}/bias', (cfg.attn_heads, hd))

    cp = 'ConditioningProcessor_0'
    dense_(cp + '/Dense_0', E, E)
    dense_(cp + '/Dense_1', E, E)
    if cfg.use_pos_emb:
        add(cp + '/pos_emb', (S, S, D))
    if cfg.use_ref_pose_emb:
        add(cp + '/ref_pose_emb_first', (D,))
        add(cp + '/ref_pose_emb_other', (D,))
    for i in range(L):
        conv(cp + f'/Conv_{i}', D, E)
    conv('Conv_0', 3, cfg.ch)

    n_xb = n_rb = 0
    res, c = S, cfg.ch
    skip_c = [c]

    def xblock(cin, feat, r):
        nonlocal n_xb
        name = f'XUNetBlock_{n_xb}'
        n_xb += 1
        resblock(name + '/ResnetBlock_0', cin, feat)
        if r in cfg.attn_resolutions:
            attnblock(name + '/AttnBlock_0', feat)
            attnblock(name + '/AttnBlock_1', feat)

    def rblock(cch):
        nonlocal n_rb
        resblock(f'ResnetBlock_{n_rb}', cch, cch)
        n_rb += 1

    for i in range(L):
        feat = cfg.ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks):
            xblock(c, feat, res)
            c = feat
            skip_c.append(c)
        if i != L - 1:
            rblock(c)
            res //= 2
            skip_c.append(c)
    xblock(c, cfg.ch * cfg.ch_mult[L - 1], res)
    c = cfg.ch * cfg.ch_mult[L - 1]
    for i in reversed(range(L)):
        feat = cfg.ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks + 1):
            xblock(c + skip_c.pop(), feat, res)
            c = feat
        if i != 0:
            rblock(c)
            res *= 2
    assert not skip_c
    gn('GroupNorm_0', c)
    conv('Conv_1', c, 3)
    return out


def param_count(cfg: RefConfig, S: int) -> int:
    return sum(int(np.prod(s)) for s in param_shapes(cfg, S).values())


def _is_zero_init(name: str) -> bool:
    """out_init_scale() kernels: every ResnetBlock's Conv_1 and the top-level Conv_1 (model/xunet.py:85-89,276-280).
    'ConditioningProcessor_0/Conv_1/kernel' (the level-1 pose-embedding conv, model/xunet.py:197-202) shares the suffix
    but is a default-initialised nn.Conv: lecun_normal."""
    return name.endswith('Conv_1/kernel') and not name.startswith('ConditioningProcessor_0/')


def nest(flat: Dict[str, torch.Tensor]) -> dict:
    tree: dict = {}
    for k, v in flat.items():
        node = tree
        parts = k.split('/')
        for part in parts[:-1]:
            node = node.setdefault(part, {})
        node[parts[-1]] = v
    return tree


def flatten(tree: dict, prefix='') -> "OrderedDict[str, torch.Tensor]":
    out = OrderedDict()
    for k, v in tree.items():
        if isinstance(v, dict):
            out.update(flatten(v, prefix + k + '/'))
        else:
            out[prefix + k] = v
    return out


def init_params(cfg: RefConfig, S: int, seed: int = 0, *, zero_init: bool = True,
                dtype=torch.float64, flat=False, bias_std: float = 0.0):
    """Flax-style initialisation (train.py:41-43): lecun_normal kernels (truncated normal, std
    sqrt(1/fan_in)/0.87962566), zero biases, GroupNorm scale 1 / bias 0, pos/ref embeddings N(0, 1/sqrt(D)).
    zero_init=False replaces the out_init_scale() zero kernels by lecun_normal so eps_hat != 0 (SURVEY F9);
    bias_std>0 additionally randomises biases / GN affine params (for stronger parity tests)."""
    g = torch.Generator().manual_seed(seed)
    flat_p = OrderedDict()
    for name, shape in param_shapes(cfg, S).items():
        leaf = name.rsplit('/', 1)[-1]
        if leaf == 'kernel':
            if zero_init and _is_zero_init(name):
                v = torch.zeros(shape, dtype=torch.float64)
            else:
                if len(shape) == 5:
                    fan_in = shape[1] * shape[2] * shape[3]
                elif len(shape) == 3:           # DenseGeneral (C, heads, hd): fan_in = C
                    fan_in = shape[0]
                else:
                    fan_in = shape[0]
                std = math.sqrt(1.0 / fan_in) / 0.87962566103423978
                v = torch.empty(shape, dtype=torch.float64)
                torch.nn.init.trunc_normal_(v, mean=0., std=1., a=-2., b=2., generator=g)
                v = v * std
        elif leaf == 'scale':
            v = torch.ones(shape, dtype=torch.float64)
            if bias_std > 0:
                v = v + bias_std * torch.randn(shape, generator=g, dtype=torch.float64)
        elif leaf == 'bias':
            v = torch.zeros(shape, dtype=torch.float64)
            if bias_std > 0:
                v = bias_std * torch.randn(shape, generator=g, dtype=torch.float64)
        else:  # pos_emb / ref_pose_emb_*
            v = torch.randn(shape, generator=g, dtype=torch.float64) / math.sqrt(POSE_EMB_DIM)
        flat_p[name] = v.to(dtype)
    return flat_p if flat else nest(flat_p)


def formula_params(cfg: RefConfig, S: int, *, dtype=torch.float64, flat=False):
    """Platform-independent non-trivial parameters (no RNG stream involved) for the committed golden vectors:
    every leaf is a scaled sinusoid of its element index; kernels have ~lecun variance, zero-init kernels are
    NOT zeroed (so eps_hat != 0), biases / GroupNorm affine are perturbed so every gradient path is exercised."""
    flat_p = OrderedDict()
    for li, (name, shape) in enumerate(param_shapes(cfg, S).items()):
        n = int(np.prod(shape))
        i = np.arange(n, dtype=np.float64)
        wave = np.sin(0.7311 * i + 1.37 * li + 0.61 * np.cos(0.0173 * i * (1 + li % 5)))
        leaf = name.rsplit('/', 1)[-1]
        if leaf == 'kernel':
            fan_in = shape[1] * shape[2] * shape[3] if len(shape) == 5 else shape[0]
            v = wave * math.sqrt(2.0 / fan_in)
        elif leaf == 'scale':
            v = 1.0 + 0.2 * wave
        elif leaf == 'bias':
            v = 0.1 * wave
        else:
            v = wave / math.sqrt(POSE_EMB_DIM)
        flat_p[name] = torch.from_numpy(v.reshape(shape)).to(dtype)
    return flat_p if flat else nest(flat_p)


# --------------------------------------------------------------------------------------
# training step (train.py:49-76)
# --------------------------------------------------------------------------------------
def loss_fn(eps_hat, noise):
    """train.py:67  jnp.mean(jnp.linalg.norm(output - noise)) == Frobenius norm of the whole residual."""
    return torch.linalg.norm((eps_hat - noise).reshape(-1))


def adam_update(p, g, m, v, step, lr=1e-4, b1=0.9, b2=0.999, eps=1e-8):
    """optax.adam (train.py:45,76): step is the 1-based count AFTER increment."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    mhat = m / (1 - b1 ** step)
    vhat = v / (1 - b2 ** step)
    return p - lr * mhat / (torch.sqrt(vhat) + eps), m, v


def loss_and_grads(params, batch, noise, cond_mask, cfg: RefConfig = SMALL, *, train=True,
                   drop_mask_fn=None, rays=None, ray_convention='v3d130_ij', emu=None):
    """apply_model (train.py:49-72) via torch autograd.  Returns (loss, flat grads dict, eps_hat)."""
    flat_p = flatten(params)
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in flat_p.items())
    eps_hat = xunet_forward(nest(leaves), batch, cond_mask, cfg, train=train, drop_mask_fn=drop_mask_fn,
                            rays=rays, ray_convention=ray_convention, emu=emu)
    loss = loss_fn(eps_hat, noise.to(eps_hat.dtype))
    grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    gd = OrderedDict()
    for (k, v), g in zip(leaves.items(), grads):
        gd[k] = torch.zeros_like(v) if g is None else g
    return loss.detach(), gd, eps_hat.detach()


# --------------------------------------------------------------------------------------
# sampler (sampling.py:16-53, 73-76, 119-151) -- schedule tables are float64 numpy in the reference
# --------------------------------------------------------------------------------------
def cosine_beta_schedule(timesteps, s=0.008):  # sampling.py:16-26
    steps = timesteps + 1
    x = np.linspace(0, timesteps, steps, dtype=np.float64)
    ac = np.cos(((x / timesteps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = 1 - (ac[1:] / ac[:-1])
    return np.clip(betas, 0, 0.9999)


def schedule_tables(T=1000):  # sampling.py:28-41
    betas = cosine_beta_schedule(T)
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.pad(ac[:-1], (1, 0), 'constant', constant_values=(1))
    post_var = betas * (1. - ac_prev) / (1. - ac)
    return dict(
        betas=betas, alphas=alphas, alphas_cumprod=ac, alphas_cumprod_prev=ac_prev,
        sqrt_alphas_cumprod=np.sqrt(ac), sqrt_one_minus_alphas_cumprod=np.sqrt(1. - ac),
        sqrt_recip_alphas_cumprod=np.sqrt(1. / ac), sqrt_recipm1_alphas_cumprod=np.sqrt(1. / ac - 1),
        posterior_variance=post_var,
        posterior_log_variance_clipped=np.log(post_var.clip(min=1e-20)),
        posterior_mean_coef1=betas * np.sqrt(ac_prev) / (1. - ac),
        posterior_mean_coef2=(1. - ac_prev) * np.sqrt(alphas) / (1. - ac))


def logsnr_schedule_cosine(t, logsnr_min=-20., logsnr_max=20.):  # sampling.py:73-76
    b = np.arctan(np.exp(-.5 * logsnr_max))
    a = np.arctan(np.exp(-.5 * logsnr_min)) - b
    return -2. * np.log(np.tan(a * t + b))


def sampler_step(eps_c, eps_u, z, time_step, noise, tab=None, w=3.0):
    """One iteration of sampling.py:128-151 given the two model outputs.  Returns (z_next, logsnr_next)."""
    tab = tab or schedule_tables()
    eps = (1 + w) * eps_c - w * eps_u                                                # :133-134
    x_recon = tab['sqrt_recip_alphas_cumprod'][time_step] * z - tab['sqrt_recipm1_alphas_cumprod'][time_step] * eps
    x_recon = torch.clamp(x_recon, -1., 1.)                                          # :137
    mean = tab['posterior_mean_coef1'][time_step] * x_recon + tab['posterior_mean_coef2'][time_step] * z
    logvar = tab['posterior_log_variance_clipped'][time_step]
    nonzero = 0.0 if time_step == 0 else 1.0                                         # :147
    z_next = mean + nonzero * math.exp(0.5 * logvar) * noise
    return z_next, float(logsnr_schedule_cosine(time_step / 1000.0))                 # :151


# --------------------------------------------------------------------------------------
# synthetic SRN-shaped inputs (dataset/data_loader.py:92-113 output contract; SURVEY 8(d))
# --------------------------------------------------------------------------------------
def _look_at(c):
    fwd = -c / np.linalg.norm(c)
    up = np.array([0., 0., 1.])
    right = np.cross(fwd, up)
    if np.linalg.norm(right) < 1e-6:
        right = np.array([1., 0., 0.])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd], axis=1)   # cam->world, columns = camera axes (x right, y down, z fwd)


def synthetic_batch(B, S, seed=1234, dtype=torch.float64):
    rng = np.random.RandomState(seed)
    tab = schedule_tables()
    x = rng.uniform(-1, 1, (B, S, S, 3))
    x0 = rng.uniform(-1, 1, (B, S, S, 3))
    noise = rng.randn(B, S, S, 3)
    t = rng.randint(0, 1000, (B,))
    z = tab['sqrt_alphas_cumprod'][t][:, None, None, None] * x0 + \
        tab['sqrt_one_minus_alphas_cumprod'][t][:, None, None, None] * noise
    logsnr = logsnr_schedule_cosine(t / 1000.0)
    Rs, ts = [], []
    for _ in range(2):
        c = rng.randn(B, 3)
        c = 1.3 * c / np.linalg.norm(c, axis=1, keepdims=True)
        Rs.append(np.stack([_look_at(ci) for ci in c]))
        ts.append(c)
    f = 131.25 * S / 128.
    K = np.tile(np.array([[f, 0, S / 2.], [0, f, S / 2.], [0, 0, 1.]])[None], (B, 1, 1))
    mk = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    batch = dict(x=mk(x), z=mk(z), logsnr=mk(logsnr), R1=mk(Rs[0]), t1=mk(ts[0]), R2=mk(Rs[1]), t2=mk(ts[1]), K=mk(K))
    return batch, mk(noise)
