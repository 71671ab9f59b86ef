"""CPU checks of the vector-Jacobian product: xunet_backward_vjp's argument errors (the library's plan is built on the host and
nothing is launched), and the fp64 reference VJP (tests/vjp_ref.py) against central finite differences."""
import ctypes as C

import pytest
import torch

from oracle import xunet_ref as R
from novel_view_synthesis_3d_b200 import _lib, XUNetConfig
from tests import vjp_ref

TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)


def _handle(lib, training):
    h = C.c_void_p()
    cs = XUNetConfig(**TINY).c_struct()
    assert lib.xunet_create(C.byref(cs), 2, 16, _lib.DTYPE_BF16, training, C.byref(h)) == 0, lib.xunet_last_error()
    return h


def _call(lib, h, d_eps=16):
    # placeholder addresses: every failing call returns before it reads or launches anything
    batch = _lib.XunetBatch(*([8] * 9), None)
    return lib.xunet_backward_vjp(h, 8, C.byref(batch), d_eps, 8, 8, 8, 0, None, None, None)


@pytest.mark.parametrize('case', ['null_d_eps', 'inference_handle', 'no_forward'])
def test_backward_vjp_rejects_bad_calls(lib, case):
    h = _handle(lib, 0 if case == 'inference_handle' else 1)
    try:
        rc = _call(lib, h, d_eps=None if case == 'null_d_eps' else 16)
        msg = lib.xunet_last_error().decode()
    finally:
        lib.xunet_destroy(h)
    assert rc != 0
    want = {'null_d_eps': 'null argument', 'inference_handle': 'training=0', 'no_forward': 'xunet_forward first'}[case]
    assert msg.startswith('xunet_backward_vjp:') and want in msg, msg


def test_reference_vjp_matches_central_differences():
    S, B = 16, 1
    cfg = R.RefConfig(**TINY)
    params = R.init_params(cfg, S, seed=3, zero_init=False, bias_std=0.1)
    batch, _ = R.synthetic_batch(B, S, seed=11)
    cond = torch.ones(B, dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    d_eps = torch.randn(B, S, S, 3, generator=g, dtype=torch.float64)
    _, gp, gx, gz = vjp_ref.vjp(params, batch, cond, d_eps, cfg)
    flat = R.flatten(params)

    def f(p=None, **inputs):
        with torch.no_grad():
            return (R.xunet_forward(R.nest(p or flat), dict(batch, **inputs), cond, cfg) * d_eps).sum().item()

    h = 1e-5
    checks = []
    for key, grad in (('x', gx), ('z', gz)):
        v = torch.randn(batch[key].shape, generator=g, dtype=torch.float64)
        fd = (f(**{key: batch[key] + h * v}) - f(**{key: batch[key] - h * v})) / (2 * h)
        checks.append((key, fd, float((grad * v).sum())))
    for name in ('Conv_0/kernel', 'XUNetBlock_1/AttnBlock_0/AttnLayer_0/DenseGeneral_0/kernel',
                 'ConditioningProcessor_0/Dense_0/kernel'):
        v = torch.randn(flat[name].shape, generator=g, dtype=torch.float64)
        fd = (f(dict(flat, **{name: flat[name] + h * v})) - f(dict(flat, **{name: flat[name] - h * v}))) / (2 * h)
        checks.append((name, fd, float((gp[name] * v).sum())))
    bad = [(k, fd, an) for k, fd, an in checks if abs(fd - an) > 1e-6 * max(abs(an), 1e-3)]
    assert not bad, bad
