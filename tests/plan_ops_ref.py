"""fp64 restatement of the conditioning, resampling, concat and loss launches, with the per-element bound each kernel is held to.

Same form as tests/launch_ref.py: |got - ref| <= rel * |ref| + floor element by element, ref the fp64 result of the values the
kernel read, the floor built from the magnitudes of what the kernel's arithmetic rounds.  The copies (concat) and the pos_emb
gradient only copy, add or round, so they are restated exactly in fp32 / bf16 (round to nearest even, as torch's casts do) and
checked for equality.  Constants are derived where they are defined.  All functions take and return float64 tensors (or the
exact fp32 / bf16 restatements) on any device.
"""
import ctypes
import math

import torch

from tests import launch_ref as L

U = L.U                 # fp32 unit roundoff 2^-24
ULP = 2. ** -23         # one fp32 ulp relative to the value (the bound of an n-ulp function is n ULP |value|)
SIN_ERR = 2. ** -22     # sinf / cosf: 2 ulp of a value of magnitude <= 1 (ulp <= 2^-24 below 1, 2^-23 at 1)
HALF_PI32 = float(torch.tensor(math.pi / 2, dtype=torch.float32))
POSE_DIM = 144


def store_rel(bf16):
    return L.store_rel(bf16)


# ======================================================================================================================
# the plan's other launches (xunet_plan_op)
# ======================================================================================================================
OP_KEY = ('kind', 'B', 'S', 'E', 'N', 'H', 'W', 'C', 'C2', 'copies', 'rs', 'fwd_pool', 'fwd_scale', 'gscale', 'bwd_pool',
          'bwd_scale', 'alpha', 'acc_x', 'acc_r', 'need_grad', 'need_grad_r', 'write_dpe', 'pos_emb', 'ref_pose_emb',
          'ray_convention')


def plan_ops(lib, cfg, B, S, dtype, training):
    """the plan's conditioning, resampling, concat, attention-residual and loss ops as dicts, in op order"""
    from novel_view_synthesis_3d_b200 import _lib
    h = ctypes.c_void_p()
    cs = cfg.c_struct()
    assert lib.xunet_create(ctypes.byref(cs), B, S, dtype, training, ctypes.byref(h)) == 0, lib.xunet_last_error()
    try:
        out = []
        for i in range(lib.xunet_plan_op_count(h)):
            r = _lib.XunetOpInfo()
            assert lib.xunet_plan_op(h, i, ctypes.byref(r)) == 0, lib.xunet_last_error()
            d = {k: getattr(r, k) for k, _ in r._fields_}
            d['copies'] = tuple(tuple(c) for c in r.copies)
            out.append(d)
        assert lib.xunet_plan_op(h, len(out), ctypes.byref(_lib.XunetOpInfo())) != 0
        return out
    finally:
        lib.xunet_destroy(h)


# ======================================================================================================================
# rounding of the fast-math helpers (common.cuh)
# ======================================================================================================================
def sigmoid(x):
    return torch.sigmoid(x)


def swish(x):
    return x * torch.sigmoid(x)


def swish_grad(x):
    s = torch.sigmoid(x)
    return s * (1. + x * (1. - s))


def swish_err(x):
    """|swishf_(x) - swish(x)| for an fp32 x.  __expf(-x) errs by 2 + floor(1.16 |x|) ulp; sigma = 1 / (1 + e) inherits
    (1 - sigma) of e's relative error; the add, __fdividef (2 ulp) and the product with x add 4 ulp:
    |swish| ((1 - sigma)(2 + 1.16 |x|) + 4) ulp.  The |x| term grows in the tail, where it is scaled by the tiny |swish|."""
    s = sigmoid(x)
    return (x * s).abs() * ((1. - s) * (2. + 1.16 * x.abs()) + 4.) * ULP


def swish_grad_err(x):
    """|swish_gradf_(x) - swish'(x)|: g = s (1 + x (1 - s)) with s = sigmoidf_(x) off by ds = s ((1 - s)(2 + 1.16 |x|) + 3) ulp
    moves g by |dg/ds| ds = |1 + x - 2 x s| ds; the four fp32 operations of g round by 4 ulp of s (1 + |x| (1 - s))."""
    s = sigmoid(x)
    ds = s * ((1. - s) * (2. + 1.16 * x.abs()) + 3.) * ULP
    return (1. + x - 2. * x * s).abs() * ds + 4. * ULP * s * (1. + x.abs() * (1. - s))


SWISH_GRAD2_MAX = 0.5   # max |swish''|: how far swish' moves when its fp32 argument rounds


def fl32(t):
    return t.to(torch.float32).to(torch.float64)


# ======================================================================================================================
# log-SNR MLP: pe = posenc_ddpm(t), h1 = pe w0 + b0, lemb = swish(h1) w1 + b1
# ======================================================================================================================
def logsnr_time(logsnr):
    """t = 1000 * 2 atan(exp(-clip(l, +-20) / 2)) / pi in fp64, of the fp32 logsnr"""
    l = logsnr.clamp(-20., 20.)
    return 1000. * 2. * torch.atan(torch.exp(-l / 2.)) / math.pi


# relative error of the fp32 argument t * f of posenc_ddpm: t takes expf, atanf (2 ulp each), the product, division by fl32(pi)
# and the product by 1000 (6 ulp together with pi's rounding); f = expf(k c) with c = fl32(-ln(10^4) / (half - 1)) takes c's
# rounding and the product k c, each 2^-24 of |k c| <= ln(10^4) = 9.21 (18.4 u), and expf's 2 ulp; the argument's own rounding
# 1 ulp.  Sum ~ 31 ulp; 2^-17 = 64 ulp holds a 2x margin.
DDPM_ARG_REL = 2. ** -17


def posenc_ddpm_check(logsnr, E):
    """(pe ref, bound) (B, E): the sin half, then the cos half, of t f_k, f_k = exp(-k ln(10^4) / (E/2 - 1)).  The argument
    errs by DDPM_ARG_REL |t f|, sinf / cosf by SIN_ERR; fp32 store."""
    half = E // 2
    t = logsnr_time(logsnr)[:, None]
    f = torch.exp(-torch.arange(half, dtype=torch.float64, device=logsnr.device) * (math.log(10000.) / (half - 1)))
    arg = t * f
    ref = torch.cat([torch.sin(arg), torch.cos(arg)], -1)
    bound = torch.cat([arg.abs(), arg.abs()], -1) * DDPM_ARG_REL + SIN_ERR + store_rel(False) * ref.abs()
    return ref, bound


def dense_check(x, w, b, x_err=None):
    """(ref, bound) of x w + b, x (B, K) the values the kernel multiplied, w (K, J), b (J): 8 fp32 fma chains of K/8 terms and
    8 adds onto the bias (acc_floor(K + 1) of sum |x||w| + |b|), x_err an absolute error of x carried by |w|, fp32 store."""
    K = x.shape[-1]
    ref = x @ w + b
    mag = x.abs() @ w.abs() + b.abs()
    bound = store_rel(False) * ref.abs() + L.acc_floor(K + 1) * mag
    if x_err is not None:
        bound = bound + x_err @ w.abs()
    return ref, bound


def logsnr_fwd_check(logsnr, w0, b0, w1, b1, pe, h1):
    """[(name, ref, bound)] chained on the kernel's own intermediates: pe, then Dense_0 on the kernel's pe, then Dense_1 on
    swish of the kernel's h1 (swishf_'s error carried by |w1|)"""
    E = w0.shape[0]
    pr, pb = posenc_ddpm_check(logsnr, E)
    hr, hb = dense_check(pe, w0, b0)
    lr, lb = dense_check(swish(h1), w1, b1, swish_err(h1))
    return [('pe', pr, pb), ('h1', hr, hb), ('lemb', lr, lb)]


def logsnr_bwd_check(dlemb, w1, pe, h1, dh1, priors=None):
    """[(name, ref, bound)] of the backward, dw0 / db0 on the kernel's own dh1.  dh1 = swish'(h1) (dlemb w1^T): a warp sums E
    products (acc_floor(E)), swish_gradf_ errs by swish_grad_err.  The weight gradients sum B products per element in fp32
    (acc_floor(B)), swish(h1) by swish_err; priors (dw0, db0, dw1, db1) are added (accumulate) with one more rounding."""
    E = w1.shape[0]
    B = dlemb.shape[0]
    g = dlemb @ w1.T
    gm = dlemb.abs() @ w1.abs().T
    sg = swish_grad(h1)
    r_dh1 = sg * g
    b_dh1 = store_rel(False) * r_dh1.abs() + sg.abs() * L.acc_floor(E) * gm + swish_grad_err(h1) * g.abs()
    out = [('dh1', r_dh1, b_dh1)]
    sw = swish(h1)
    terms = [('dw0', pe.T @ dh1, pe.abs().T @ dh1.abs(), None),
             ('db0', dh1.sum(0), dh1.abs().sum(0), None),
             ('dw1', sw.T @ dlemb, sw.abs().T @ dlemb.abs(), swish_err(h1).T @ dlemb.abs()),
             ('db1', dlemb.sum(0), dlemb.abs().sum(0), None)]
    for i, (name, r, m, extra) in enumerate(terms):
        p = priors[i] if priors is not None else None
        ref = r if p is None else p + r
        bound = store_rel(False) * ref.abs() + L.acc_floor(B) * m + (0. if extra is None else extra)
        if p is not None:
            bound = bound + U * (r.abs() + ref.abs())
        out.append((name, ref, bound))
    return out


# ======================================================================================================================
# pose embedding: rays + posenc_nerf, masks, pos_emb / ref_pose_emb
# ======================================================================================================================
def kinv_check(K):
    """(ref, bound) of K^-1 (B, 9): inverted in fp64 by the kernel (cofactors), rounded to fp32 once"""
    ref = torch.linalg.inv(K.reshape(-1, 3, 3)).reshape(-1, 9)
    return ref, 2. ** -23 * ref.abs() + 2. ** -40 * ref.abs().amax(-1, keepdim=True)


def pixel_coords(S, convention, device=None):
    """p (S, S, 3) fed to K^-1: (row + .5, col + .5, 1) (convention 0) or (col + .5, row + .5, 1) (convention 1)"""
    ii, jj = torch.meshgrid(torch.arange(S, dtype=torch.float64, device=device) + 0.5,
                            torch.arange(S, dtype=torch.float64, device=device) + 0.5, indexing='ij')
    p0, p1 = (ii, jj) if convention == 0 else (jj, ii)
    return torch.stack([p0, p1, torch.ones_like(p0)], -1)


def ray_dirs(kinv, R, S, convention):
    """(dir ref, dir bound) (B, S, S, 3) of normalize(R K^-1 p) from the fp32 K^-1 the kernel read.  In fp32 c = K^-1 p and
    w = R c are 3-term dot products, each ~3 roundings: 6 u of |R| |K^-1| |p| on w (x2 margin: 12 u); dividing by |w| doubles
    a relative error of w at most, and the norm, the reciprocal and the product add ~4 u (8 u)."""
    ki = kinv.reshape(-1, 3, 3)
    p = pixel_coords(S, convention, kinv.device)
    c = torch.einsum('bij,hwj->bhwi', ki, p)
    w = torch.einsum('bij,bhwj->bhwi', R, c)
    wm = torch.einsum('bij,bhwj->bhwi', R.abs(), torch.einsum('bij,hwj->bhwi', ki.abs(), p))
    n = torch.linalg.norm(w, dim=-1, keepdim=True)
    d = w / n
    return d, 2. * 12. * U * torch.linalg.norm(wm, dim=-1, keepdim=True) / n + 8. * U


def posenc_nerf32(v, nd):
    """posenc_nerf(v, 0, nd) (..., 3 + 6 nd) in fp64 at the kernel's fp32 arguments: v, sin(fl32(2^k v)),
    sin(fl32(fl32(2^k v) + fl32(pi/2))), the channels scale-major (3 per scale)"""
    v32 = v.to(torch.float32)
    xb = torch.cat([v32 * (2. ** k) for k in range(nd)], -1)
    sh = xb + torch.tensor(HALF_PI32, dtype=torch.float32, device=v.device)
    return torch.cat([v32.double(), torch.sin(xb.double()), torch.sin(sh.double())], -1)


def posenc_nerf_exact(v, v_err, nd):
    """(ref, bound) of posenc_nerf(v, 0, nd) from an fp64 v known to v_err: the channels sin(2^k v) and
    cos(2^k v) = sin(2^k v + pi/2) move by 2^k v_err; the fp32 add of pi/2 rounds by 2^-24 (2^k |v| + pi/2); sinf: SIN_ERR"""
    sc = torch.cat([torch.full_like(v, 2. ** k) for k in range(nd)], -1)
    xb = torch.cat([v * (2. ** k) for k in range(nd)], -1)
    ve = torch.cat([v_err.expand_as(v)] * nd, -1)
    ref = torch.cat([v, torch.sin(xb), torch.cos(xb)], -1)
    e = sc * ve
    bound = torch.cat([v_err.expand_as(v), e + SIN_ERR, e + U * (xb.abs() + 2.) + SIN_ERR], -1)
    return ref, bound


def pose_emb_check(dtype, R1, t1, R2, t2, kinv, cond, S, convention, pos_emb=None, ref_first=None, ref_other=None, rays=None,
                   dirs32=None):
    """(ref, bound) (2B, S, S, 144) of the stored pose embedding.  Origin channels: at the fp32 camera centre (or the explicit
    ray origin), exact arguments, SIN_ERR.  Direction channels: explicit rays at their fp32 components; generated rays at the
    kernel's own fp32 directions dirs32 (B, 2, S, S, 3) when given (fp32 plans export them), else from fp64 rays (ray_dirs,
    posenc_nerf_exact).  Masked samples are 0.  pos_emb and ref add two fp32 roundings 2^-23 (|s| + |pos_emb| + |ref|),
    then the store."""
    B = cond.shape[0]
    dev = cond.device
    embs, errs = [], []
    for f, (R, t) in enumerate(((R1, t1), (R2, t2))):
        if rays is not None:
            pos, d = rays[:, f, ..., :3], rays[:, f, ..., 3:]
            pe_pos = posenc_nerf32(pos, 15)
            pe_dir = posenc_nerf32(d, 8)
            e_pos = torch.full_like(pe_pos, SIN_ERR)
            e_pos[..., :3] = 0.
            e_dir = torch.full_like(pe_dir, SIN_ERR)
            e_dir[..., :3] = 0.
        else:
            pe_pos = posenc_nerf32(t, 15)[:, None, None, :].expand(B, S, S, 93)
            e_pos = torch.full_like(pe_pos, SIN_ERR)
            e_pos[..., :3] = 0.
            if dirs32 is not None:
                pe_dir = posenc_nerf32(dirs32[:, f], 8)
                e_dir = torch.full_like(pe_dir, SIN_ERR)
                e_dir[..., :3] = 0.
            else:
                d, de = ray_dirs(kinv, R, S, convention)
                pe_dir, e_dir = posenc_nerf_exact(d, de, 8)
        embs.append(torch.cat([pe_pos, pe_dir], -1))
        errs.append(torch.cat([e_pos, e_dir], -1))
    m = (cond != 0).double().reshape(B, 1, 1, 1, 1)
    s = (torch.stack(embs, 1) * m).reshape(2 * B, S, S, POSE_DIM)
    err = (torch.stack(errs, 1) * m).reshape(2 * B, S, S, POSE_DIM)
    ref, mag = s.clone(), s.abs()
    if pos_emb is not None:
        ref, mag = ref + pos_emb, mag + pos_emb.abs()
    if ref_first is not None:
        rf = torch.stack([ref_first, ref_other]).repeat(B, 1)[:, None, None, :]
        ref, mag = ref + rf, mag + rf.abs()
    bound = err + (2. ** -23 * mag if (pos_emb is not None or ref_first is not None) else 0.) + store_rel(dtype == 1) * ref.abs()
    return ref, bound


def pose_emb_added(dtype, base32, pos_emb32, ref_first32, ref_other32):
    """the stored embedding with pos_emb and ref added, exactly, from the fp32 embedding base32 (2B, S, S, 144) the kernel
    formed without them: fl32(fl32(base + pos_emb) + ref), then the store (masked samples: base = 0)"""
    v = base32
    if pos_emb32 is not None:
        v = v + pos_emb32
    if ref_first32 is not None:
        B = base32.shape[0] // 2
        v = v + torch.stack([ref_first32, ref_other32]).repeat(B, 1)[:, None, None, :]
    return v.to(torch.bfloat16 if dtype == 1 else torch.float32)


def pose_emb_bwd_exact(dpose, prior=None):
    """the exact fp32 pos_emb gradient: per element s0 = sum over frames 0, s1 over frames 1 (fp32, in sample order), s0 + s1,
    then += prior when accumulating.  dpose (2B, S, S, 144) as stored (fp32 or bf16)."""
    d = dpose.to(torch.float32)
    s0 = torch.zeros_like(d[0])
    s1 = torch.zeros_like(d[0])
    for b in range(d.shape[0] // 2):
        s0 = s0 + d[2 * b]
        s1 = s1 + d[2 * b + 1]
    g = s0 + s1
    return g if prior is None else prior + g, s0, s1


def pose_emb_ref_check(s, prior):
    """(ref, bound) of dref_* (144) += the sum of the fp32 per-pixel sums s (S, S, 144) over pixels: fp64 atomics (2^-40 of
    the magnitudes), then two fp32 roundings (the sum, the add to the prior)"""
    r = s.double().reshape(-1, POSE_DIM).sum(0)
    m = s.double().abs().reshape(-1, POSE_DIM).sum(0)
    ref = prior + r
    return ref, U * (r.abs() + ref.abs()) + 2. ** -40 * m


# ======================================================================================================================
# FiLM embedding: semb = swish(lemb[b] + pe)
# ======================================================================================================================
def _emb_arg(lemb, pe):
    """x = lemb[n / 2] + pe (N, HW, E) and the rounding of its fp32 add"""
    N = pe.shape[0]
    x = pe + lemb.repeat_interleave(2, 0)[:N, None, :]
    return x, U * x.abs()


def film_emb_check(lemb, pe, bf16):
    x, xe = _emb_arg(lemb, pe)
    ref = swish(x)
    # |swish'| <= 1.1
    return ref, store_rel(bf16) * ref.abs() + swish_err(x) + 1.1 * xe


def film_emb_bwd_check(lemb, pe, dsemb, bf16, dlemb_prior):
    """(dpe ref, dpe bound, dlemb ref, dlemb bound).  dz = dsemb swish'(x): swish_gradf_'s error and the argument's rounding
    (|swish''| <= 1/2), one product rounding; dlemb (B, E) = prior + the sum of dz over the 2 HW pixels of a sample: fp32
    partial sums per thread (acc_floor of the pixel count), fp64 across threads, two roundings at the fold."""
    x, xe = _emb_arg(lemb, pe)
    dz = dsemb * swish_grad(x)
    dz_err = dsemb.abs() * (swish_grad_err(x) + SWISH_GRAD2_MAX * xe) + U * dz.abs()
    b_dpe = store_rel(bf16) * dz.abs() + dz_err
    N, HW, E = pe.shape
    P = 2 * HW
    s = dz.reshape(N // 2, P, E).sum(1)
    m = dz.abs().reshape(N // 2, P, E).sum(1)
    e = dz_err.reshape(N // 2, P, E).sum(1)
    ref = dlemb_prior + s
    return dz, b_dpe, ref, e + L.acc_floor(P) * m + U * (s.abs() + ref.abs())


# ======================================================================================================================
# resample, channel copies, scale-add
# ======================================================================================================================
def resample(x, pool):
    """(N, H, W, C): pool -> the 2x2 sum (N, H/2, W/2, C); else each pixel repeated 2x2 (N, 2H, 2W, C)"""
    N, H, W, C = x.shape
    if pool:
        return x.reshape(N, H // 2, 2, W // 2, 2, C).sum((2, 4))
    return x[:, :, None, :, None, :].expand(N, H, 2, W, 2, C).reshape(N, 2 * H, 2 * W, C)


def resample_check(x, pool, scale, bf16, prior=None):
    """(ref, bound) of scale * resample(x) (+ prior): one rounding per operation -- three adds of the 2x2 sum, the product
    by scale, the add of the prior (which nvcc may contract into an fma: fewer roundings) -- 2^-24 of the magnitudes each;
    then the store"""
    r = scale * resample(x, pool)
    m = abs(scale) * resample(x.abs(), pool)
    ref = r if prior is None else prior + r
    bound = store_rel(bf16) * ref.abs() + (3. if pool else 0.) * U * m + U * r.abs()
    if prior is not None:
        bound = bound + U * ref.abs()
    return ref, bound


def copy_channels_exact(src, dst, Cs, Cd, src_off, dst_off, Cc, accumulate):
    """the exact result of a channel copy on (npix, Cs) / (npix, Cd) tensors of the storage dtype: copied, or added in fp32 and
    rounded to the storage type; the other channels of dst unchanged"""
    out = dst.clone()
    s = src[:, src_off:src_off + Cc]
    if accumulate:
        s = (s.to(torch.float32) + dst[:, dst_off:dst_off + Cc].to(torch.float32)).to(dst.dtype)
    out[:, dst_off:dst_off + Cc] = s
    return out


def scale_add_check(src, alpha, bf16, prior=None):
    """(ref, bound) of alpha src (+ prior): the product, the add (or one fma), the store"""
    r = alpha * src
    ref = r if prior is None else prior + r
    bound = store_rel(bf16) * ref.abs() + U * r.abs()
    if prior is not None:
        bound = bound + U * ref.abs()
    return ref, bound


# ======================================================================================================================
# loss = ||eps - noise||, dO frame 1 = (eps - noise) / loss
# ======================================================================================================================
def loss_check(eps, noise, bf16):
    """(sumsq ref, bound, loss ref, bound, dO ref (2B, S, S, 3), bound).  The fp32 difference rounds (2 u on its square); the
    sum of squares runs as fp32 fma chains per thread, warp and 8-lane shuffles (acc_floor of the count), fp64 across blocks,
    one rounding at the fold; sqrtf adds u and halves the sum's relative error; dO = r / loss rounds r, loss and the
    division.  Loss 0: dO is exactly 0."""
    B = eps.shape[0]
    r = eps - noise
    n = r.numel()
    ss = (r * r).sum()
    ss_rel = 2. * U + L.acc_floor(n) + U
    loss = torch.sqrt(ss)
    loss_rel = ss_rel / 2. + U
    g = r / loss if float(loss) > 0 else torch.zeros_like(r)
    dO = torch.zeros((2 * B,) + tuple(r.shape[1:]), dtype=torch.float64, device=r.device)
    dO[1::2] = g
    dO_b = store_rel(bf16) * dO.abs()
    dO_b[1::2] += g.abs() * (U + loss_rel + U)
    return ss, ss_rel * ss, loss, loss_rel * loss, dO, dO_b
