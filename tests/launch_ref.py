"""fp64 restatement of the convolution and attention launches, with the per-element bound each kernel is held to.

Every check has the form |got - ref| <= rel * |ref| + floor, element by element: ref is the fp64 result of the kernel's own
inputs (the values it read, as fp64), rel covers the final rounding to the storage type, and the floor is the error of the
kernel's arithmetic, built from the magnitudes of the terms it sums.  The constants are derived where they are defined.

Layouts are the kernels': activations channels-last (N, H, W, C); a conv weight is the flat Flax leaf order
[seg][tap][ci][segw] (nseg > 1 only for the fused q|k|v projection, whose three Dense kernels lie end to end); attention reads
qkv (N, L, 3C) = [q | k | v], heads of hd = C / heads channels, and with cross the keys and values of frame n ^ 1.
All functions take and return float64 tensors on any device.
"""
import ctypes
import math

import torch

# ======================================================================================================================
# the plans bench.py measures, and their launches as the plan reports them (xunet_plan_launch)
# ======================================================================================================================
# name -> (preset, side, xunet_create batch, dtype (0 fp32, 1 bf16), training).  small64 / small128 train at B = 8, full64 /
# full128 at B = 4; the full128 sampler runs 1 and 4 views in flight, and Sampler evaluates the conditional and unconditional
# halves of classifier-free guidance as one forward, so its engine has batch 2 x views; the fp32 verify mode at B = 2.
PLANS = {
    'small64': ('SMALL', 64, 8, 1, 1),
    'small128': ('SMALL', 128, 8, 1, 1),
    'full64': ('FULL_3DIM', 64, 4, 1, 1),
    'full128': ('FULL_3DIM', 128, 4, 1, 1),
    'sampler1': ('FULL_3DIM', 128, 2, 1, 0),
    'sampler4': ('FULL_3DIM', 128, 8, 1, 0),
    'small64_f32': ('SMALL', 64, 2, 0, 1),
}
CONV_KEY = ('N', 'Hi', 'Wi', 'Ci', 'Ho', 'Wo', 'Co', 'ksize', 'stride', 'nseg', 'residual', 'alpha', 'fwd', 'dgrad', 'wgrad',
            'emits_stats', 'bwd_alpha', 'accumulate', 'gn_mode')
ATTN_KEY = ('N', 'L', 'C', 'heads', 'cross', 'impl', 'emits_stats')


def plan_launches(lib, cfg, B, S, dtype, training):
    """(launches as dicts in op order, leaf names in leaf order) of the plan of (cfg, B, S, dtype, training)"""
    from novel_view_synthesis_3d_b200 import _lib
    h = ctypes.c_void_p()
    cs = cfg.c_struct()
    assert lib.xunet_create(ctypes.byref(cs), B, S, dtype, training, ctypes.byref(h)) == 0, lib.xunet_last_error()
    try:
        out = []
        for i in range(lib.xunet_plan_launch_count(h)):
            r = _lib.XunetLaunchInfo()
            assert lib.xunet_plan_launch(h, i, ctypes.byref(r)) == 0, lib.xunet_last_error()
            out.append({k: getattr(r, k) for k, _ in r._fields_})
        assert lib.xunet_plan_launch(h, len(out), ctypes.byref(_lib.XunetLaunchInfo())) != 0
        names = []
        name, ndim, shape, off = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_longlong * 5)(), ctypes.c_longlong()
        for i in range(lib.xunet_param_leaves(h)):
            assert lib.xunet_param_leaf(h, i, ctypes.byref(name), ctypes.byref(ndim), ctypes.byref(shape), ctypes.byref(off)) == 0
            names.append(name.value.decode())
        return out, names
    finally:
        lib.xunet_destroy(h)


def plan_config(cfg):
    """a plan's model configuration: a preset's name (PLANS) or an XUNetConfig"""
    import novel_view_synthesis_3d_b200 as P
    return getattr(P, cfg) if isinstance(cfg, str) else cfg


def launch_key(dtype, training, r):
    """what changes a launch: two launches with one key run the same kernels on the same shapes and arguments"""
    return (r['kind'], dtype) + (tuple(r[k] for k in CONV_KEY) if r['kind'] == 0 else (training,) + tuple(r[k] for k in ATTN_KEY))


def unique_launches(lib, plans=PLANS, exclude=None):
    """every launch of `plans` (name -> (preset name or XUNetConfig, side, batch, dtype, training)) once, deduplicated by what
    changes the launch: [(id, dtype, training, launch)], the id naming the first plan and leaf (conv) or attention index that
    has it.  Launches that the plans of `exclude` also have are left out.  An attention's backward runs in training plans
    only."""
    seen, out = set(), []
    if exclude is not None:
        seen.update(launch_key(dtype, training, r) for _, dtype, training, r in unique_launches(lib, exclude))
    for plan, (cfg, S, B, dtype, training) in plans.items():
        launches, names = plan_launches(lib, plan_config(cfg), B, S, dtype, training)
        na = 0
        for r in launches:
            key = launch_key(dtype, training, r)
            if r['kind'] == 1:
                na += 1
            if key in seen:
                continue
            seen.add(key)
            where = names[r['leaf']].replace('/kernel', '') if r['kind'] == 0 else f'attn{na - 1}'
            out.append((f'{plan}:{where}', dtype, training, r))
    return out


# ======================================================================================================================
# rounding constants
# ======================================================================================================================
U = 2. ** -24            # fp32 unit roundoff
# bf16 keeps 8 significand bits: rounding to nearest errs by at most 2^-8 of the value
BF16_OP = 2. ** -8        # one rounding of an operand to bf16 (P before PV, dS before dS K)
# a stored result: one bf16 rounding (2^-8 relative; the fp32 work before it is in the floors, which hold a 5x margin for the
# (1 + 2^-8) it is scaled by); fp32: the store and the epilogue's operations, a few 2^-24 relative: 2^-21
BF_REL = 2. ** -8
F32_REL = 2. ** -21


def acc_floor(K):
    """Coefficient of sum|terms| for an fp32 sum of K products (wgmma or fma chains).  Each addition rounds the partial sum by
    at most 2^-24 of it (twice that if the adder truncates), and the K errors take random signs: a random walk of
    sqrt(K) 2^-24 sum|terms|.  2^-16 at K = 2304 (9 taps x 256 channels), i.e. 5.3 sqrt(K) 2^-24, keeps a 5x margin over it
    for every K: 2^-14.5 at K = 9 x 2048, the widest reduction of the full model, 2^-19.6 at K = 16, a head_dim-16 score.
    Where the terms share a sign (inputs with offsets) the tensor cores' accumulator, which truncates, errs by up to about
    (K / 16) 2^-24 sum|terms| (one rounding per 16-product wgmma step) instead, which reaches this floor near K = 2^13 terms
    per CTA: same-signed inputs summed 2^14 pixels per CTA measured 1.5 x over it.  The weight-gradient kernels never split a
    sum into longer runs than on the whole device (wgrad_tc's split-K factor, common.cuh xu_num_sms), whose per-CTA runs stay
    within it on the benchmarked plans.  The closest call an H100 measured there, err / bound 0.93, is the weight gradient of
    a strided pose-embedding conv."""
    return 2. ** -16 * math.sqrt(K / 2304.)


def store_rel(bf16):
    return BF_REL if bf16 else F32_REL


def excess(got, ref, bound):
    """(worst (|got - ref|) / bound, the flat index where it occurs, number of elements over their bound).  A NaN result is
    over its bound (and the worst)."""
    err = (got.double() - ref).abs()
    r = err / bound.clamp_min(1e-300)
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), i, int((~(err <= bound)).sum())


def within(got, ref, bound):
    return excess(got, ref, bound)[2] == 0


# ======================================================================================================================
# convolution: y = alpha * (sum_{tap, ci} x[pixel (+) tap] W[tap][ci][co] + bias + res), SAME padding, stride s
# ======================================================================================================================
def same_pad(n, ks, stride):
    """(low padding, output size) of Flax's SAME padding"""
    out = (n + stride - 1) // stride
    return max((out - 1) * stride + ks - n, 0) // 2, out


def weight(w_flat, ks, Ci, Co, nseg=1):
    """flat Flax leaf order [seg][tap][ci][segw] -> (taps, Ci, Co)"""
    taps = ks * ks
    return w_flat.reshape(nseg, taps, Ci, Co // nseg).permute(1, 2, 0, 3).reshape(taps, Ci, Co)


def weight_flat(w, nseg=1):
    """inverse of weight(): (taps, Ci, Co) -> flat Flax leaf order"""
    taps, Ci, Co = w.shape
    return w.reshape(taps, Ci, nseg, Co // nseg).permute(2, 0, 1, 3).reshape(-1)


def _windows(x, ks, stride, Ho, Wo):
    """the input window of every tap: x padded SAME, one (N, Ho, Wo, Ci) slice per tap (dy, dx) in tap order"""
    N, Hi, Wi, Ci = x.shape
    ph, _ = same_pad(Hi, ks, stride)
    pw, _ = same_pad(Wi, ks, stride)
    hp = (Ho - 1) * stride + ks
    wp = (Wo - 1) * stride + ks
    xp = torch.zeros(N, hp, wp, Ci, dtype=x.dtype, device=x.device)
    h1, w1 = min(Hi, hp - ph), min(Wi, wp - pw)
    xp[:, ph:ph + h1, pw:pw + w1] = x[:, :h1, :w1]
    for dy in range(ks):
        for dx in range(ks):
            yield xp[:, dy:dy + (Ho - 1) * stride + 1:stride, dx:dx + (Wo - 1) * stride + 1:stride]


def conv(x, w, ks, stride=1):
    """x (N, Hi, Wi, Ci), w (taps, Ci, Co) -> (N, Ho, Wo, Co), no bias"""
    N, Hi, Wi, Ci = x.shape
    _, Ho = same_pad(Hi, ks, stride)
    _, Wo = same_pad(Wi, ks, stride)
    y = torch.zeros(N, Ho, Wo, w.shape[-1], dtype=x.dtype, device=x.device)
    for t, win in enumerate(_windows(x, ks, stride, Ho, Wo)):
        y += win @ w[t]
    return y


def conv_dgrad(dy, w, ks, stride, Hi, Wi):
    """adjoint of conv() in x: dy (N, Ho, Wo, Co) -> (N, Hi, Wi, Ci)"""
    N, Ho, Wo, Co = dy.shape
    Ci = w.shape[1]
    ph, _ = same_pad(Hi, ks, stride)
    pw, _ = same_pad(Wi, ks, stride)
    hp, wp = (Ho - 1) * stride + ks, (Wo - 1) * stride + ks
    dxp = torch.zeros(N, max(hp, ph + Hi), max(wp, pw + Wi), Ci, dtype=dy.dtype, device=dy.device)
    for t in range(ks * ks):
        dyy, dxx = divmod(t, ks)
        dxp[:, dyy:dyy + (Ho - 1) * stride + 1:stride, dxx:dxx + (Wo - 1) * stride + 1:stride] += dy @ w[t].T
    return dxp[:, ph:ph + Hi, pw:pw + Wi].contiguous()


def conv_wgrad(x, dy, ks, stride):
    """gradient in w: (taps, Ci, Co) = sum over output pixels of window(x) (x) dy"""
    N, Ho, Wo, Co = dy.shape
    d2 = dy.reshape(-1, Co)
    return torch.stack([win.reshape(-1, x.shape[-1]).T @ d2 for win in _windows(x, ks, stride, Ho, Wo)])


def conv_fwd_check(x, w, bias, res, alpha, ks, stride, bf16):
    """(ref, bound) of the stored forward output.  x: the stored input; w (taps, Ci, Co): the weights the kernel multiplies
    (the bf16 shadow on the tensor cores, the fp32 master weights on the SIMT and direct kernels); res may be None.
    Floor: acc_floor(taps Ci) of sum|x||w| + |bias| + |res| (the epilogue's two adds and the alpha product round within it)."""
    K = ks * ks * x.shape[-1]
    ref = conv(x, w, ks, stride) + bias
    mag = conv(x.abs(), w.abs(), ks, stride) + bias.abs()
    if res is not None:
        ref, mag = ref + res, mag + res.abs()
    ref, mag = alpha * ref, abs(alpha) * mag
    return ref, store_rel(bf16) * ref.abs() + acc_floor(K) * mag


def conv_dgrad_check(dy, w, alpha, ks, stride, Hi, Wi, bf16, prior=None):
    """(ref, bound) of the stored data gradient alpha * W^T dy (+ prior when the launch accumulates).  Each dx element sums
    taps x Co products.  An accumulating launch rounds twice on the tensor cores (the epilogue's bf16 tile, then the bf16 add of
    the TMA reduce-add at L2) and once on the SIMT kernel: rel (|delta| + |ref|) covers 2^-8 |delta| + 2^-8 |prior + delta|."""
    K = ks * ks * w.shape[-1]
    delta = alpha * conv_dgrad(dy, w, ks, stride, Hi, Wi)
    mag = abs(alpha) * conv_dgrad(dy.abs(), w.abs(), ks, stride, Hi, Wi)
    rel = store_rel(bf16)
    if prior is None:
        return delta, rel * delta.abs() + acc_floor(K) * mag
    ref = prior + delta
    return ref, rel * (delta.abs() + ref.abs()) + acc_floor(K) * mag


def conv_wgrad_check(x, dy, alpha, ks, stride, dw_prior, db_prior):
    """(ref_dw, bound_dw, ref_db, bound_db) of the weight and bias gradients ADDED to the fp32 priors: dW[tap][ci][co] +=
    alpha sum_pixels window(x)[ci] dy[co], dbias += alpha sum_pixels dy.  The kernels sum their share of the pixels in fp32
    (at most all N Ho Wo of them: acc_floor of that count bounds every split), the shares in fp64, and round fp64 -> fp32 once
    when the sum is added to the prior (2^-24 |ref|, 2^-23 with the add)."""
    N, Ho, Wo, Co = dy.shape
    K = N * Ho * Wo
    dw = alpha * conv_wgrad(x, dy, ks, stride)
    dwm = abs(alpha) * conv_wgrad(x.abs(), dy.abs(), ks, stride)
    db = alpha * dy.reshape(-1, Co).sum(0)
    dbm = abs(alpha) * dy.abs().reshape(-1, Co).sum(0)
    rdw, rdb = dw_prior + dw, db_prior + db
    return rdw, 2. ** -23 * rdw.abs() + acc_floor(K) * dwm, rdb, 2. ** -23 * rdb.abs() + acc_floor(K) * dbm


# ======================================================================================================================
# attention over frames: out = (softmax(q k^T / sqrt(hd)) v + res) / sqrt(2), lse = log sum exp(q k^T / sqrt(hd))
# ======================================================================================================================
def split_heads(qkv, heads, cross):
    """qkv (N, L, 3C) -> q, k, v (N, heads, L, hd); with cross, frame n attends to the keys and values of frame n ^ 1"""
    N, L, C3 = qkv.shape
    C = C3 // 3
    q, k, v = (t.reshape(N, L, heads, C // heads).permute(0, 2, 1, 3) for t in torch.split(qkv, C, dim=-1))
    if cross:
        perm = torch.arange(N, device=qkv.device) ^ 1
        k, v = k[perm], v[perm]
    return q, k, v


def _merge(t):
    """(N, heads, L, hd) -> (N, L, C)"""
    N, h, L, hd = t.shape
    return t.permute(0, 2, 1, 3).reshape(N, L, h * hd)


def _p_error(q, k, t, base):
    """relative error bound of each probability exp(t - base) as the kernels form it, t = q.k / sqrt(hd) the scaled score:
    the fp32 score sums hd products (scale acc_floor(hd) sum|q||k|); the exponent argument t log2e - base is formed by one fma
    with a rounded scale and a rounded base (2 roundings of |t| and |base|, x2 margin: 4 u); ex2.approx / __expf err by 2^-22
    plus 2 u |argument|, covered by 2^-21"""
    hd = q.shape[-1]
    scale = 1. / math.sqrt(hd)
    ds = acc_floor(hd) * scale * (q.abs() @ k.abs().transpose(-1, -2))
    return ds + 4. * U * (t.abs() + base.abs()) + 2. ** -21


def attn_fwd_check(qkv, res, heads, cross, bf16=True):
    """(out, out_bound, lse, lse_bound).  out per element:
      - the rounding of P to bf16 before the PV product: 2^-8 sum_k P|v| (l sums the unrounded P);
      - the probability errors e_k (_p_error), which move out by sum_k P e_k (v_k - o): <= sum P e |v| + (sum P e) |o|;
      - the fp32 PV sum and row sum l over L keys: acc_floor(L) (sum P|v| + |o|) (the per-block rescales, L/64 products, fit in);
      - the epilogue (o / l + res) / sqrt2: 4 u (|o| + |res|), then the store (BF_REL; fp32: F32_REL).
    fp32 (bf16=False): P is not rounded before the product (u instead of 2^-8).
    lse per row, absolute: sum P e + acc_floor(L) (the relative error of l) + 2^-20 (__logf, 2^-21.4 absolute) + 4 u |lse|
    (the base-2 max times ln2 and the final add)."""
    q, k, v = split_heads(qkv, heads, cross)
    N, h, L, hd = q.shape
    t = (q @ k.transpose(-1, -2)) / math.sqrt(hd)
    lse = torch.logsumexp(t, dim=-1)
    mx = t.amax(-1, keepdim=True)
    P = torch.exp(t - lse[..., None])
    e = _p_error(q, k, t, mx)
    o = P @ v
    pv = P @ v.abs()
    pe = (P * e).sum(-1, keepdim=True)
    err_o = ((BF16_OP if bf16 else U) + acc_floor(L)) * pv + (P * e) @ v.abs() + (pe + acc_floor(L)) * o.abs()
    o, err_o = _merge(o), _merge(err_o)
    out = (o + res) / math.sqrt(2.)
    out_b = store_rel(bf16) * out.abs() + (err_o + 4. * U * (o.abs() + res.abs())) / math.sqrt(2.)
    lse_b = pe[..., 0] + acc_floor(L) + 2. ** -20 + 4. * U * (lse.abs() + mx[..., 0].abs())
    return out, out_b, lse, lse_b


def attn_bwd_check(qkv, res, out, dout, lse, heads, cross, bf16=True):
    """(dqkv ref, dqkv bound) on the kernel's own inputs: the stored out and lse.  As the kernels form them: P = exp(t - lse),
    O = out sqrt2 - res, dO = dout / sqrt2, D = rowsum(dO O), dP = dO v^T, dS = P (dP - D) / sqrt(hd); dQ = dS k, dK = dS^T q,
    dV = P^T dO (dK, dV of frame n ^ 1 under cross).  Error of dS per (query, key):
      scale P (e |dP - D| + acc_floor(hd) (sum|dO||v| + sum|dO| (sqrt2 |out| + |res|))) + 4 u |dS|
    (e the probability error with lse as the base; D's fp32 fma chain also rounds O's formation, 2 u per term, inside the
    acc_floor).  Then dQ sums dS |k| with dS rounded to bf16 (2^-8 |dS|) and fp32 sums of at most L terms (acc_floor(L)):
      dQ: (2^-8 + acc_floor(L)) sum_k |dS||k| + sum_k err(dS)|k|;   dK likewise over queries with |q|;
      dV: (2^-8 + acc_floor(L)) sum_q P|dO| + sum_q P e |dO|   (P rounded to bf16);
    each + BF_REL of the stored value.  fp32 (bf16=False): no operand rounding (u instead of 2^-8), F32_REL stores."""
    q, k, v = split_heads(qkv, heads, cross)
    N, h, L, hd = q.shape
    C = h * hd
    scale = 1. / math.sqrt(hd)
    sp = lambda a: a.reshape(N, L, h, hd).permute(0, 2, 1, 3)
    O = sp(out * math.sqrt(2.) - res)
    Omag = sp(out.abs() * math.sqrt(2.) + res.abs())
    dO = sp(dout) / math.sqrt(2.)
    t = (q @ k.transpose(-1, -2)) * scale
    base = lse[..., None]
    P = torch.exp(t - base)
    e = _p_error(q, k, t, base)
    D = (dO * O).sum(-1, keepdim=True)
    dP = dO @ v.transpose(-1, -2)
    dS = P * (dP - D) * scale
    dmag = acc_floor(hd) * (dO.abs() @ v.abs().transpose(-1, -2) + (dO.abs() * Omag).sum(-1, keepdim=True))
    err_ds = scale * P * (e * (dP - D).abs() + dmag) + 4. * U * dS.abs()
    cl = (BF16_OP if bf16 else U) + acc_floor(L)
    dq = dS @ k
    dq_b = cl * (dS.abs() @ k.abs()) + err_ds @ k.abs()
    dk = dS.transpose(-1, -2) @ q
    dk_b = cl * (dS.abs().transpose(-1, -2) @ q.abs()) + err_ds.transpose(-1, -2) @ q.abs()
    dv = P.transpose(-1, -2) @ dO
    dv_b = cl * (P.transpose(-1, -2) @ dO.abs()) + (P * e).transpose(-1, -2) @ dO.abs()
    if cross:   # keys and values of query frame n belong to frame n ^ 1
        perm = torch.arange(N, device=qkv.device) ^ 1
        dk, dk_b, dv, dv_b = dk[perm], dk_b[perm], dv[perm], dv_b[perm]
    ref = torch.cat([_merge(dq), _merge(dk), _merge(dv)], -1)
    bound = store_rel(bf16) * ref.abs() + torch.cat([_merge(dq_b), _merge(dk_b), _merge(dv_b)], -1)
    return ref, bound


def attn_qkv(N, L, C, heads, peaked, g):
    """attention inputs (N, L, 3C): per-channel offsets on q, k and v, and per-frame offsets on v, so that a routing error
    between frames, heads or channels shows.  peaked: the scores grow from key block to key block (a 64-key ramp along one
    direction u per head), with a step of 6 / sqrt(hd) u before the last block, so that every query's largest score lies in the
    last 64-key block (a partial one when L % 64 != 0) and the online softmax rescales its state on the way there."""
    hd = C // heads
    nb = (L + 63) // 64
    ch = torch.arange(3 * C, dtype=torch.float64)
    fr = torch.arange(N, dtype=torch.float64)[:, None, None]
    if not peaked:
        x = torch.randn(N, L, 3 * C, generator=g, dtype=torch.float64) + 0.1 * torch.cos(ch)
        x[..., 2 * C:] += 0.2 * fr
        return x
    u = torch.randint(0, 2, (heads, hd), generator=g).double() * 2. - 1.
    amp = 12. / math.sqrt(hd)
    blk = torch.arange(L) // 64
    ramp = torch.where(blk == nb - 1, torch.tensor(1.), 0.5 * blk.double() / max(nb - 1, 1))   # 0 .. 0.5, then 1
    x = 0.1 * torch.randn(N, L, 3 * C, generator=g, dtype=torch.float64) + 0.02 * torch.cos(ch)
    x[..., :C] += amp * u.reshape(-1)
    x[..., C:2 * C] += ramp[:, None] * u.reshape(-1)
    x[..., 2 * C:] += torch.randn(N, L, C, generator=g, dtype=torch.float64) + 0.2 * fr
    return x


def attn_bwd_exact(qkv, res, dout, heads, cross):
    """dqkv of the exact fp64 forward (autograd): the chain check of the whole backward from the bf16 inputs"""
    x = qkv.detach().clone().requires_grad_(True)
    q, k, v = split_heads(x, heads, cross)
    p = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1]), dim=-1)
    out = (_merge(p @ v) + res) / math.sqrt(2.)
    out.backward(dout)
    return x.grad
