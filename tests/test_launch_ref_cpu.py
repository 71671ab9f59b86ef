"""CPU checks of tests/launch_ref.py, the fp64 references and per-element bounds the conv and attention launches are held to:
the references against torch, the bounds accepting a result that carries nothing but its final bf16 rounding, and rejecting
each of a set of subtle kernel bugs."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import launch_ref as L

F64 = torch.float64


def _bf(t):
    return t.to(torch.bfloat16).to(F64)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _conv_torch(x, w, ks, stride):
    """Flax SAME conv by torch.nn.functional.conv2d with explicit asymmetric padding"""
    N, H, W, Ci = x.shape
    ph, Ho = L.same_pad(H, ks, stride)
    pw, Wo = L.same_pad(W, ks, stride)
    eh, ew = max((Ho - 1) * stride + ks - H, 0) - ph, max((Wo - 1) * stride + ks - W, 0) - pw
    xp = F.pad(x.permute(0, 3, 1, 2), (pw, ew, ph, eh))
    wt = w.reshape(ks, ks, Ci, -1).permute(3, 2, 0, 1)
    return F.conv2d(xp, wt, stride=stride).permute(0, 2, 3, 1)


@pytest.mark.parametrize('N,H,W,Ci,Co,ks,stride', [(2, 8, 8, 16, 24, 3, 1), (2, 8, 8, 5, 7, 3, 2), (4, 16, 16, 6, 8, 3, 8),
                                                   (2, 6, 10, 8, 12, 1, 1)])
def test_conv_reference_and_its_gradients_match_torch(N, H, W, Ci, Co, ks, stride):
    g = _g(1)
    x = torch.randn(N, H, W, Ci, generator=g, dtype=F64, requires_grad=True)
    w = torch.randn(ks * ks, Ci, Co, generator=g, dtype=F64, requires_grad=True)
    y = L.conv(x, w, ks, stride)
    ref = _conv_torch(x, w, ks, stride)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)
    dy = torch.randn(ref.shape, generator=g, dtype=F64)
    gx, gw = torch.autograd.grad(ref, (x, w), dy)
    assert torch.allclose(L.conv_dgrad(dy, w.detach(), ks, stride, H, W), gx, rtol=1e-12, atol=1e-12)
    assert torch.allclose(L.conv_wgrad(x.detach(), dy, ks, stride), gw, rtol=1e-12, atol=1e-12)


def test_segmented_weight_layout():
    """the q|k|v projection: three (Ci, segw) kernels end to end give output channels [q | k | v]"""
    g = _g(2)
    Ci, segw = 4, 6
    ws = [torch.randn(Ci, segw, generator=g, dtype=F64) for _ in range(3)]
    flat = torch.cat([w.reshape(-1) for w in ws])
    w = L.weight(flat, 1, Ci, 3 * segw, 3)
    assert torch.equal(w[0], torch.cat(ws, 1))
    assert torch.equal(L.weight_flat(w, 3), flat)


# ======================================================================================================================
# conv: bf16(ref) is accepted, the mutations are not
# ======================================================================================================================
def _conv_case(seed, N=2, H=8, W=8, Ci=16, Co=24, ks=3, nseg=1, residual=True, alpha=1 / math.sqrt(2)):
    g = _g(seed)
    x = _bf(torch.randn(N, H, W, Ci, generator=g, dtype=F64) + 0.3 * torch.arange(N, dtype=F64)[:, None, None, None])
    w = _bf(torch.randn(ks * ks, Ci, Co, generator=g, dtype=F64) / math.sqrt(ks * ks * Ci))
    b = 0.3 * torch.randn(Co, generator=g, dtype=F64)
    res = _bf(torch.randn(N, H, W, Co, generator=g, dtype=F64)) if residual else None
    return x, w, b, res, alpha


def test_conv_forward_accepts_its_rounding():
    x, w, b, res, alpha = _conv_case(3)
    ref, bound = L.conv_fwd_check(x, w, b, res, alpha, 3, 1, True)
    assert L.within(_bf(ref), ref, bound)
    ref32, bound32 = L.conv_fwd_check(x, w, b, res, alpha, 3, 1, False)
    assert L.within(ref32.float(), ref32, bound32)


def test_conv_forward_rejects_a_dropped_tap_at_a_border_pixel():
    x, w, b, res, alpha = _conv_case(4)
    ref, bound = L.conv_fwd_check(x, w, b, res, alpha, 3, 1, True)
    # output pixel (0, 0) of frame 1 loses tap (2, 2), which reads input pixel (1, 1)
    got = ref.clone()
    got[1, 0, 0] -= alpha * (x[1, 1, 1] @ w[8])
    assert not L.within(_bf(got), ref, bound)


def test_conv_forward_rejects_a_padding_shift_in_one_row():
    x, w, b, res, alpha = _conv_case(5)
    ref, bound = L.conv_fwd_check(x, w, b, res, alpha, 3, 1, True)
    # row 3 of frame 0 reads its input one column to the left: the padding column moves from the left edge to the right
    xs = torch.zeros_like(x)
    xs[:, :, 1:] = x[:, :, :-1]
    shifted = alpha * (L.conv(xs, w, 3) + b + res)
    got = ref.clone()
    got[0, 3] = shifted[0, 3]
    assert not L.within(_bf(got), ref, bound)


def test_conv_forward_rejects_swapped_qkv_segments_in_one_channel_block():
    x, w, b, _, _ = _conv_case(6, Ci=32, Co=3 * 32, ks=1, nseg=3, residual=False)
    ref, bound = L.conv_fwd_check(x, w, b, None, 1., 1, 1, True)
    # the first 8-channel block of the q and k segments trade places
    got = ref.clone()
    got[..., 0:8], got[..., 32:40] = ref[..., 32:40], ref[..., 0:8]
    assert not L.within(_bf(got), ref, bound)


def test_accumulating_dgrad_accepts_its_two_roundings_and_rejects_an_overwrite():
    g = _g(7)
    N, H, W, Ci, Co = 2, 8, 8, 16, 24
    dy = _bf(torch.randn(N, H, W, Co, generator=g, dtype=F64))
    w = _bf(torch.randn(9, Ci, Co, generator=g, dtype=F64) / math.sqrt(9 * Co))
    prior = _bf(torch.randn(N, H, W, Ci, generator=g, dtype=F64))
    ref, bound = L.conv_dgrad_check(dy, w, 0.5, 3, 1, H, W, True, prior=prior)
    delta = ref - prior
    # the tensor-core path: the tile rounded to bf16, then added to the bf16 prior by the TMA unit (rounded again)
    assert L.within(_bf(prior + _bf(delta)), ref, bound)
    assert not L.within(_bf(delta), ref, bound)        # the prior overwritten instead of added to
    # and without accumulation: one rounding
    ref0, bound0 = L.conv_dgrad_check(dy, w, 0.5, 3, 1, H, W, True)
    assert L.within(_bf(ref0), ref0, bound0)
    assert not L.within(_bf(ref0 + prior), ref0, bound0)   # added to a destination it should have overwritten


def test_wgrad_accepts_an_fp32_result():
    g = _g(8)
    x = _bf(torch.randn(4, 8, 8, 16, generator=g, dtype=F64))
    dy = _bf(torch.randn(4, 8, 8, 32, generator=g, dtype=F64))
    dw0, db0 = torch.randn(9, 16, 32, generator=g, dtype=F64).float().double(), torch.randn(32, generator=g, dtype=F64)
    rdw, bdw, rdb, bdb = L.conv_wgrad_check(x, dy, 0.7, 3, 1, dw0, db0)
    assert L.within(rdw.float(), rdw, bdw) and L.within(rdb.float(), rdb, bdb)
    # one tap's gradient missing is far outside
    got = rdw.clone()
    got[4] -= 0.7 * L.conv_wgrad(x, dy, 3, 1)[4]
    assert not L.within(got.float(), rdw, bdw)


# ======================================================================================================================
# attention
# ======================================================================================================================
def _attn_case(seed, peaked, N=4, Lk=128, C=32, heads=2):
    g = _g(seed)
    qkv = _bf(L.attn_qkv(N, Lk, C, heads, peaked, g))
    res = _bf(torch.randn(N, Lk, C, generator=g, dtype=F64) + 0.3 * torch.arange(N, dtype=F64)[:, None, None])
    return qkv, res


@pytest.mark.parametrize('heads,hd', [(2, 16), (1, 64), (2, 128)])
def test_peaked_inputs_put_every_largest_score_in_the_last_key_block(heads, hd):
    g = _g(9)
    Lk = 256
    q, k, _ = L.split_heads(L.attn_qkv(2, Lk, heads * hd, heads, True, g), heads, 1)
    s = q @ k.transpose(-1, -2)
    assert bool((s.argmax(-1) >= Lk - 64).all())
    # and the block maxima rise from block to block for most queries: the online softmax rescales on the way
    bm = s.reshape(*s.shape[:-1], Lk // 64, 64).amax(-1)
    assert float((bm[..., 1:] > bm[..., :-1]).double().mean()) > 0.9


@pytest.mark.parametrize('peaked', [False, True])
@pytest.mark.parametrize('cross', [0, 1])
def test_attention_forward_accepts_its_rounding_and_rejects_a_skipped_key_block(peaked, cross):
    qkv, res = _attn_case(10, peaked)
    heads = 2
    out, out_b, lse, lse_b = L.attn_fwd_check(qkv, res, heads, cross)
    q, k, v = L.split_heads(qkv, heads, cross)
    sdpa = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(out.shape)
    assert torch.allclose(out, (sdpa + res) / math.sqrt(2.), rtol=1e-12, atol=1e-12)
    assert torch.allclose(lse, torch.logsumexp((q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1]), -1), rtol=1e-12)
    assert L.within(_bf(out), out, out_b) and L.within(lse.float(), lse, lse_b)
    # query tile 1 (queries 64..127) of frame 2, head 1 never sees one key block: block 0 of the moderate input (about half
    # the mass), the last block of the peaked one.  A peaked input's early blocks hold less than e^-6 of the mass, below the
    # 2^-8 of the bf16 store: skipping one of them cannot be told apart from rounding.
    t = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    blk = slice(64, 128) if peaked else slice(0, 64)
    t[2, 1, 64:, blk] = -math.inf
    p = torch.softmax(t, -1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(out.shape)
    bad = (o + res) / math.sqrt(2.)
    got = out.clone()
    got[2, 64:, 16:] = bad[2, 64:, 16:]
    bad_lse = lse.clone()
    bad_lse[2, 1, 64:] = torch.logsumexp(t[2, 1, 64:], -1)
    assert not L.within(_bf(got), out, out_b)
    assert not L.within(bad_lse.float(), lse, lse_b)


def _bwd_case(seed, peaked, cross):
    qkv, res = _attn_case(seed, peaked)
    g = _g(seed + 1)
    out, _, lse, _ = L.attn_fwd_check(qkv, res, 2, cross)
    out, lse = _bf(out), lse.float().double()               # what the forward stored: the backward's inputs
    dout = _bf(torch.randn(out.shape, generator=g, dtype=F64) + 0.1 * torch.arange(out.shape[-1], dtype=F64) / 32)
    return qkv, res, out, lse, dout


@pytest.mark.parametrize('cross', [0, 1])
def test_attention_backward_reference_is_the_gradient(cross):
    """with the exact forward's out and lse as inputs the reference is autograd's gradient"""
    qkv, res = _attn_case(11, False)
    out, _, lse, _ = L.attn_fwd_check(qkv, res, 2, cross)
    dout = torch.randn(out.shape, generator=_g(12), dtype=F64)
    ref, _ = L.attn_bwd_check(qkv, res, out, dout, lse, 2, cross)
    assert torch.allclose(ref, L.attn_bwd_exact(qkv, res, dout, 2, cross), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize('peaked', [False, True])
@pytest.mark.parametrize('cross', [0, 1])
def test_attention_backward_accepts_its_rounding_and_rejects_subtle_bugs(peaked, cross):
    qkv, res, out, lse, dout = _bwd_case(13, peaked, cross)
    heads, C = 2, 32
    hd = C // heads
    ref, bound = L.attn_bwd_check(qkv, res, out, dout, lse, heads, cross)
    assert L.within(_bf(ref), ref, bound)
    # dV of head 1 without the 1/sqrt2 of dO
    got = ref.clone()
    got[..., 2 * C + hd:] *= math.sqrt(2.)
    assert not L.within(_bf(got), ref, bound)
    # one dS term (the largest) missing from one dQ element: frame 1, head 0, query 5, channel 3
    q, k, v = L.split_heads(qkv, heads, cross)
    sp = lambda a: a.reshape(*a.shape[:2], heads, hd).permute(0, 2, 1, 3)
    P = torch.exp((q @ k.transpose(-1, -2)) / math.sqrt(hd) - lse[..., None])
    dO = sp(dout) / math.sqrt(2.)
    D = (dO * sp(out * math.sqrt(2.) - res)).sum(-1, keepdim=True)
    dS = P * (dO @ v.transpose(-1, -2) - D) / math.sqrt(hd)
    terms = dS[1, 0, 5] * k[1, 0, :, 3]
    j = int(terms.abs().argmax())
    got = ref.clone()
    got[1, 5, 3] -= terms[j]
    assert not L.within(_bf(got), ref, bound)
