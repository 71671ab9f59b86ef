"""The tensor-core attention backward as two atomic-free passes (a dQ kernel over query tiles, then a dK/dV kernel over key
tiles): gradients against an fp64 restatement, bit-identical repeats, and a scratch buffer written only in its D rows."""
import math

import pytest
import torch

from tests.util import rel_l2

pytestmark = pytest.mark.gpu

# N, L, C, heads, cross  ->  head_dim 16 / 32 / 64 / 128, self and cross attention, L = 128 and 1024
CASES = [(2, 128, 32, 2, 0), (4, 1024, 64, 4, 1), (2, 128, 64, 2, 1), (2, 1024, 64, 2, 0),
         (2, 128, 128, 2, 0), (2, 1024, 128, 2, 1), (2, 128, 256, 2, 1), (2, 1024, 128, 1, 0)]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _problem(lib, case):
    N, L, Cc, heads, cross = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFF)
    qkv = (torch.randn(N, L, 3 * Cc, generator=g, dtype=torch.float32) * 1.5).to(torch.bfloat16).cuda()
    res = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16).cuda()
    dout = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16).cuda()
    out = torch.zeros(N, L, Cc, dtype=torch.bfloat16, device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_attention(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), lse.data_ptr(), N, L, Cc, heads, cross,
                                  _stream()) == 0, lib.xunet_last_error()
    return qkv, res, dout, out, lse


def _bwd(lib, case, prob, scratch):
    N, L, Cc, heads, cross = case
    qkv, res, dout, out, lse = prob
    dqkv = torch.full((N, L, 3 * Cc), float('nan'), dtype=torch.bfloat16, device='cuda')
    rc = lib.xunet_op_attention_bwd(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                    scratch.data_ptr(), dqkv.data_ptr(), N, L, Cc, heads, cross, _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    return dqkv


def _reference_grads(case, prob):
    N, L, Cc, heads, cross = case
    hd = Cc // heads
    qkv, res, dout = (t.cpu().double() for t in prob[:3])
    qr = qkv.requires_grad_(True)
    q, k, v = [t.reshape(N, L, heads, hd) for t in torch.split(qr, Cc, dim=-1)]
    if cross:
        perm = torch.arange(N) ^ 1
        k, v = k[perm], v[perm]
    w = torch.softmax(torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k), dim=-1)
    o = torch.einsum('nhqk,nkhd->nqhd', w, v).reshape(N, L, Cc)
    ((o + res) / math.sqrt(2)).backward(dout)
    return qr.grad


@pytest.mark.parametrize('case', CASES)
def test_split_backward_is_exact_and_bit_reproducible(lib, case):
    N, L, Cc, heads, cross = case
    prob = _problem(lib, case)
    scratch = torch.empty(N * heads * L, dtype=torch.float32, device='cuda')
    first = _bwd(lib, case, prob, scratch)
    second = _bwd(lib, case, prob, scratch)
    assert torch.equal(first, second)                                  # no atomics: the same bits on every call
    ref = _reference_grads(case, prob)
    errs = [rel_l2(a.float().cpu(), b) for a, b in zip(torch.split(first, Cc, dim=-1), torch.split(ref, Cc, dim=-1))]
    assert max(errs) < 4e-2, errs


@pytest.mark.parametrize('case', CASES)
def test_split_backward_writes_only_the_d_rows_of_its_scratch(lib, case):
    """dscratch needs N*heads*L floats (D = rowsum(dO * O)); a larger buffer keeps everything past them untouched."""
    N, L, Cc, heads, cross = case
    prob = _problem(lib, case)
    nd = N * heads * L
    scratch = torch.full((N * L * (heads + Cc),), float('nan'), dtype=torch.float32, device='cuda')
    dqkv = _bwd(lib, case, prob, scratch)
    assert bool(torch.isnan(scratch[nd:]).all())
    assert torch.equal(dqkv, _bwd(lib, case, prob, torch.empty(nd, dtype=torch.float32, device='cuda')))
    _, res, dout, out, _ = (t.cpu().double() for t in prob)
    hd = Cc // heads
    D = ((dout / math.sqrt(2)) * (out * math.sqrt(2) - res)).reshape(N, L, heads, hd).sum(-1).permute(0, 2, 1).reshape(-1)
    assert rel_l2(scratch[:nd].cpu(), D) < 1e-5


@pytest.mark.parametrize('case', [CASES[0], CASES[1], CASES[5]])
def test_split_backward_hands_a_zeroed_scratch_back_zeroed(lib, case, monkeypatch):
    """XUNET_OP_ATTN_FOLD=1: the caller's all-zero scratch comes back all-zero, with the same gradients as without it."""
    N, L, Cc, heads, cross = case
    prob = _problem(lib, case)
    plain = _bwd(lib, case, prob, torch.empty(N * heads * L, dtype=torch.float32, device='cuda'))
    monkeypatch.setenv('XUNET_OP_ATTN_FOLD', '1')
    scratch = torch.zeros(N * L * (heads + Cc), dtype=torch.float32, device='cuda')
    for _ in range(2):
        assert torch.equal(_bwd(lib, case, prob, scratch), plain)
        assert float(scratch.abs().max()) == 0.0
