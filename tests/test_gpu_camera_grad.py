"""The camera gradient of the vector-Jacobian product (xunet_backward_vjp_inputs, Engine.backward_vjp_inputs,
XUNet.vjp(camera_grads=True), XUNet.apply_autograd with camera leaves) on the GPU: the ray-gradient kernels alone against fp64
from the engine's own inputs, parity of dR / dt / dK (or the rays) with autograd through the fp64 oracle, the bf16 noise floor,
and the contracts (cond_mask zeros, unchanged parameter / view gradients, fixed bits, graph replay, errors, autograd)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from oracle import xunet_ref as R
from tests import camera_grad_ref as CG
from tests.util import np_batch, rel_l2, to_ref_cfg

pytestmark = pytest.mark.gpu

SMALL = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4, dropout=0.0)
TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)


def _d_eps(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, S, S, 3, generator=g, dtype=torch.float32).cuda()


def _cond(B):
    return np.array(([1.0, 0.0, 1.0] * B)[:B], np.float32)


def _explicit_rays(batch, S, conv):
    """(B,2,S,S,6) fp32 rays of the batch's cameras, slightly perturbed so that they are not the library's own."""
    r = [R.camera_rays(batch[rk], batch[tk], batch['K'], S, S, conv) for rk, tk in (('R1', 't1'), ('R2', 't2'))]
    rays = torch.stack([torch.cat([p, d], -1) for p, d in r], 1)
    g = torch.Generator().manual_seed(2)
    return (rays + 1e-2 * torch.randn(rays.shape, generator=g, dtype=torch.float64)).float()


def _components(cfgd, B, S, nb, conv, rays):
    """The fp32 ray components the engine's posenc used: the given rays, or the generated ones read back from the raw-x
    channels of an fp32 forward's posenc tensor (the same ray code as the bf16 one)."""
    if rays is not None:
        r = rays.double().numpy()
        return r[..., :3], r[..., 3:]
    m = P.XUNet(**cfgd, dtype='fp32', ray_convention=conv)
    eng = m.engine(B, S, False)
    eng.load_inputs(nb, cond_mask=np.ones(B, np.float32))
    eng.forward(m.init({'params': 0}, {'x': np.zeros((B, S, S, 3))})['params'].flat, train=False)
    pe = eng.read_tap('pose_emb').double().cpu().numpy().reshape(B, 2, S, S, 144)
    return pe[..., 0:3], pe[..., 93:96]


# ---- 1. the ray-gradient kernels alone ----------------------------------------------------------------------------------------
KERNEL_CASES = [  # S, levels, emb_ch, B, ray convention, explicit rays
    (16, 4, 32, 1, 'v3d130_ij', False),
    (16, 2, 256, 3, 'opencv_uv', True),
    (32, 2, 256, 3, 'opencv_uv', True),
    (32, 4, 1024, 1, 'v3d130_ij', False),
    (64, 4, 1024, 3, 'v3d130_ij', True),
    (64, 2, 32, 3, 'opencv_uv', False),
    (128, 1, 32, 1, 'opencv_uv', False),
    (128, 4, 256, 1, 'v3d130_ij', False),
]


@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
@pytest.mark.parametrize('S,levels,E,B,conv,explicit', KERNEL_CASES)
def test_ray_gradient_kernel_matches_fp64_conv_transpose(dtype, S, levels, E, B, conv, explicit):
    cfgd = dict(ch=32, ch_mult=(1,) * levels, emb_ch=E, num_res_blocks=1, attn_resolutions=(), attn_heads=4, dropout=0.0)
    model = P.XUNet(**cfgd, dtype=dtype, ray_convention=conv)
    flat = model.init({'params': 3}, {'x': np.zeros((B, S, S, 3))}, zero_init=False)['params'].flat
    eng = model.engine(B, S, True)
    batch, _ = R.synthetic_batch(B, S, seed=11)
    nb = np_batch(batch)
    cond = _cond(B)
    rays = _explicit_rays(batch, S, conv) if explicit else None
    eng.load_inputs(nb, cond_mask=cond)
    eng.set_rays(rays)
    eng.forward(flat, train=False)
    eng.set_rays(None)
    _, out = eng.backward_vjp_inputs(flat, _d_eps(B, S, 13), rays=True)
    torch.cuda.synchronize()
    got = out['rays'].double().cpu().numpy()
    want = CG.d_rays_ref(eng, flat, _components(cfgd, B, S, nb, conv, rays), cond, dtype == 'bf16')
    tol = 1e-5 if dtype == 'bf16' else 1e-6
    assert np.all(got[cond == 0] == 0.0)
    got_t, want_t = torch.from_numpy(got), torch.from_numpy(want)
    assert rel_l2(got_t, want_t) < tol, rel_l2(got_t, want_t)
    border = torch.ones(S, S, dtype=torch.bool)
    border[1:-1, 1:-1] = False
    assert rel_l2(got_t[:, :, border], want_t[:, :, border]) < tol


# ---- 2./3. parity with autograd through the fp64 oracle -----------------------------------------------------------------------
def _parity(dtype, explicit):
    S, B = 64, 2
    model = P.XUNet(**SMALL, dtype=dtype)
    rcfg = to_ref_cfg(model.config)
    ref_params = R.init_params(rcfg, S, seed=7, zero_init=False, bias_std=0.1)
    eng = model.engine(B, S, True)
    flat = model.flat_from_tree(ref_params, S, B)
    batch, _ = R.synthetic_batch(B, S, seed=1234)
    cond = np.array([1.0, 1.0], np.float32)
    rays = _explicit_rays(batch, S, 'v3d130_ij') if explicit else None
    eng.load_inputs(np_batch(batch), cond_mask=cond)
    eng.set_rays(rays)
    eng.forward(flat, train=False)
    eng.set_rays(None)
    d_eps = _d_eps(B, S, 9)
    _, out = eng.backward_vjp_inputs(flat, d_eps, rays=explicit, cameras=not explicit)
    torch.cuda.synchronize()
    keys = ('rays',) if explicit else CG.CAMERA_KEYS
    got = {k: out[k].double().cpu() for k in keys}
    rr = None if rays is None else tuple((rays[:, f, ..., :3].double(), rays[:, f, ..., 3:].double()) for f in range(2))
    args = (ref_params, batch, torch.from_numpy(cond).double(), d_eps.double().cpu(), rcfg)
    return got, args, rr


@pytest.mark.parametrize('explicit', [False, True], ids=['cameras', 'rays'])
def test_fp32_camera_gradients_match_the_reference(explicit):
    got, args, rr = _parity('fp32', explicit)
    ref = CG.camera_vjp(*args, rays=rr)
    rel = {k: rel_l2(got[k], ref[k]) for k in ref}
    print(f'fp32 camera gradients: rel-L2 {rel}')
    assert max(rel.values()) < 2e-3, rel


@pytest.mark.parametrize('explicit', [False, True], ids=['cameras', 'rays'])
def test_bf16_camera_gradients_sit_on_the_bf16_noise_floor(explicit):
    got, args, rr = _parity('bf16', explicit)
    exact = CG.camera_vjp(*args, rays=rr)
    emu = CG.camera_vjp(*args, rays=rr, emu=CG.PoseSTE())
    ratios = {k: rel_l2(got[k], exact[k]) / rel_l2(emu[k], exact[k]) for k in exact}
    print(f'bf16 camera gradients: engine/floor ratios {ratios}')
    assert max(ratios.values()) < 3.0, ratios


# ---- 4. contracts -----------------------------------------------------------------------------------------------------------
def _setup(dtype, B=3, S=16, cond=None):
    model = P.XUNet(**dict(TINY, dropout=0.1), dtype=dtype)
    flat = model.init({'params': 3}, {'x': np.zeros((B, S, S, 3))}, zero_init=False)['params'].flat
    eng = model.engine(B, S, True)
    batch, _ = R.synthetic_batch(B, S, seed=21)
    nb = np_batch(batch)
    eng.load_inputs(nb, cond_mask=_cond(B) if cond is None else cond)
    torch.cuda.synchronize()
    return model, flat, eng, batch, nb


def _bits(t):
    return t.clone().view(torch.int32)


@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_camera_outputs_change_nothing_else_and_repeat_bit_for_bit(dtype):
    model, flat, eng, _, _ = _setup(dtype)
    d_eps = _d_eps(3, 16, 23)
    eng.forward(flat, train=True, seed=5)
    g, dx, dz = eng.backward_vjp(flat, d_eps, dx=True, dz=True)
    base = [_bits(t) for t in (g, dx, dz)]
    runs = []
    for _ in range(2):
        eng.forward(flat, train=True, seed=5)
        g2, out = eng.backward_vjp_inputs(flat, d_eps, dx=True, dz=True, cameras=True)
        torch.cuda.synchronize()
        assert all(torch.equal(a, _bits(b)) for a, b in zip(base, (g2, out['x'], out['z'])))
        runs.append({k: _bits(v) for k, v in out.items()})
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])
    # cond_mask = 0 (sample 1): exact zeros in every camera output; the others are not all zero
    for k in ('rays',) + CG.CAMERA_KEYS:
        v = runs[0][k].view(torch.float32)
        assert bool((v[1] == 0).all()) and bool((v[0] != 0).any()) and bool((v[2] != 0).any()), k
    # the generated-ray reduction equals the numpy restatement of it applied to the engine's d_rays
    rays = runs[0]['rays'].view(torch.float32).double().cpu().numpy()
    inp = {k: eng.inp[k].double().cpu().numpy() for k in CG.CAMERA_KEYS}
    ref = CG.camera_reduce(rays, (inp['R1'], inp['R2']), inp['K'], 16)
    for k in CG.CAMERA_KEYS:
        got = runs[0][k].view(torch.float32).double().cpu().numpy()
        assert np.abs(got - ref[k]).max() <= 1e-5 * np.abs(ref[k]).max(), k


@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_graph_replay_gives_the_eager_camera_bits(dtype):
    model, flat, eng, _, _ = _setup(dtype)
    d_eps = _d_eps(3, 16, 29)
    eng.forward(flat, train=True, seed=5)
    _, out = eng.backward_vjp_inputs(flat, d_eps, dx=True, cameras=True)
    torch.cuda.synchronize()
    eager = {k: v.clone() for k, v in out.items()}
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        eng.forward(flat, train=True, seed=5)
        eng.backward_vjp_inputs(flat, d_eps, dx=True, cameras=True)
        stream.synchronize()
        with torch.cuda.graph(graph, stream=stream):
            eng.forward(flat, train=True, seed=5)
            eng.backward_vjp_inputs(flat, d_eps, dx=True, cameras=True)
    torch.cuda.synchronize()
    for v in out.values():
        v.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(out[k], eager[k]) for k in eager)


def test_camera_gradient_errors_are_rejected():
    model, flat, eng, batch, nb = _setup('bf16', B=2, cond=np.ones(2, np.float32))
    d_eps = _d_eps(2, 16, 31)
    eng.forward(flat, train=False)
    lib = _lib.load()
    dR = torch.zeros(2, 3, 3, device='cuda')
    d_rays = torch.zeros(2, 2, 16, 16, 6, device='cuda')

    def call(ig, rays=None):
        cb = _lib.XunetBatch.from_buffer_copy(eng.cbatch)
        cb.rays = rays
        return lib.xunet_backward_vjp_inputs(eng.h, flat.data_ptr(), C.byref(cb), d_eps.data_ptr(), eng.seed.data_ptr(),
                                             eng.ws.data_ptr(), eng.grads.data_ptr(), 0, C.byref(ig), None)

    assert call(_lib.XunetInputGrads(dR1=dR.data_ptr())) != 0
    assert 'd_rays' in lib.xunet_last_error().decode()
    assert call(_lib.XunetInputGrads(d_rays=d_rays.data_ptr(), dR1=dR.data_ptr()), rays=d_rays.data_ptr()) != 0
    assert 'rays' in lib.xunet_last_error().decode()
    assert call(_lib.XunetInputGrads(d_rays=d_rays.data_ptr()), rays=d_rays.data_ptr()) == 0
    torch.cuda.synchronize()
    # Python: camera gradients of a forward that was given explicit rays
    eng.set_rays(_explicit_rays(batch, 16, 'v3d130_ij'))
    eng.forward(flat, train=False)
    eng.set_rays(None)
    with pytest.raises(ValueError):
        eng.backward_vjp_inputs(flat, d_eps, cameras=True)


@pytest.mark.parametrize('explicit', [False, True], ids=['cameras', 'rays'])
def test_autograd_camera_grads_equal_vjp_fn_bit_for_bit(explicit):
    S, B = 16, 2
    model, flat0, eng, batch, nb = _setup('bf16', B=B, cond=np.array([1.0, 0.0], np.float32))
    cond = np.array([1.0, 0.0], np.float32)
    rays = _explicit_rays(batch, S, 'v3d130_ij').cuda() if explicit else None
    loss = lambda eps: (eps * eps).sum()
    cams = {k: torch.from_numpy(nb[k]).float().cuda().requires_grad_(True) for k in CG.CAMERA_KEYS}
    ray_leaf = rays.clone().requires_grad_(True) if explicit else None
    flat = flat0.detach().clone().requires_grad_(True)
    eps = model.apply_autograd(flat, dict(nb, **cams), cond_mask=cond, train=False, rays=ray_leaf)
    loss(eps).backward()

    eps2, vjp_fn = model.vjp({'params': model.tree_from_flat(flat0, S, B)}, nb, cond_mask=cond, train=False, rays=rays,
                             camera_grads=True)
    assert torch.equal(eps.detach(), eps2)
    e = eps2.clone().requires_grad_(True)
    d_eps, = torch.autograd.grad(loss(e), e)
    tree, inputs = vjp_fn(d_eps.contiguous())
    assert torch.equal(flat.grad, tree.flat)
    if explicit:
        assert torch.equal(ray_leaf.grad, inputs['rays']) and bool((ray_leaf.grad != 0).any())
        assert all(cams[k].grad is None for k in CG.CAMERA_KEYS)
    else:
        for k in CG.CAMERA_KEYS:
            assert torch.equal(cams[k].grad, inputs[k]) and bool((cams[k].grad != 0).any()), k
    # a forward in between is refused
    eps = model.apply_autograd(flat, dict(nb, **cams), cond_mask=cond, train=False, rays=ray_leaf)
    eng.forward(flat0, train=False)
    with pytest.raises(RuntimeError):
        loss(eps).backward()
