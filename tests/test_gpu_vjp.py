"""The vector-Jacobian product of the forward (xunet_backward_vjp, Engine.backward_vjp, XUNet.vjp, XUNet.apply_autograd) on
the GPU: bit identity with the two built-in losses when seeded with their output gradients, fp32 and bf16 parity of every
gradient with the fp64 reference (tests/vjp_ref.py), the input-gradient kernel alone against fp64, finite differences on the
engine itself, determinism and graph replay, the gradient-bucket hook, and the Python surface."""
import math

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from oracle import xunet_ref as R
from tests import vjp_ref
from tests.util import np_batch, rel_l2, to_ref_cfg

pytestmark = pytest.mark.gpu

TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)
SMALL = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4, dropout=0.0)
WIDE = dict(ch=256, ch_mult=(1,), emb_ch=32, num_res_blocks=1, attn_resolutions=(), attn_heads=4, dropout=0.0)


def _setup(cfgd, dtype, B, S, seed=21, cond=None):
    """A training engine of a fresh model with non-zero-init weights, loaded with a synthetic batch and its noise."""
    model = P.XUNet(**cfgd, dtype=dtype)
    flat = model.init({'params': 3}, {'x': np.zeros((B, S, S, 3))}, zero_init=False)['params'].flat
    eng = model.engine(B, S, True)
    batch, noise = R.synthetic_batch(B, S, seed=seed)
    cond = np.array(([1.0, 0.0] * B)[:B], np.float32) if cond is None else cond
    eng.load_inputs(np_batch(batch), cond_mask=cond, noise=noise.numpy())
    torch.cuda.synchronize()
    return model, flat, eng, batch, noise.numpy().astype(np.float32)


def _d_eps(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, S, S, 3, generator=g, dtype=torch.float32).cuda()


def _vjp(eng, flat, d_eps, seed=5, train=True, **kw):
    eng.forward(flat, train=train, seed=seed)
    g, dx, dz = eng.backward_vjp(flat, d_eps, dx=True, dz=True, **kw)
    torch.cuda.synchronize()
    return g.clone(), dx.clone(), dz.clone()


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- 1. bit identity with the built-in losses --------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_seeded_with_the_loss_gradients_it_equals_the_built_in_losses(dtype):
    S, B = 16, 3
    model, flat, eng, batch, noise = _setup(dict(TINY, dropout=0.1), dtype, B, S, cond=np.array([1.0, 0.0, 1.0], np.float32))
    per = S * S * 3
    c = np.float32(2.0 / (B * per))

    def mse_seed(eps):
        return torch.from_numpy(c * (eps - noise)).cuda()                  # float32 subtraction and product, rounded once each

    def fixed(seed, **kw):
        eps = eng.forward(flat, train=True, seed=seed).cpu().numpy()
        loss, g = eng.backward(flat, **kw)
        torch.cuda.synchronize()
        return eps, float(loss), g.clone()

    # weighted-MSE seed
    eps, _, g_mse = fixed(5, loss='mse')
    g, _, _ = _vjp(eng, flat, mse_seed(eps), seed=5)
    assert bool((g_mse != 0).any()) and _bits_equal(g, g_mse)
    # Frobenius seed: fl32((eps - noise) / loss) with the loss the engine returned
    eps, loss, g_frob = fixed(5)
    d = torch.from_numpy((eps - noise) / np.float32(loss)).cuda()
    g, _, _ = _vjp(eng, flat, d, seed=5)
    assert _bits_equal(g, g_frob)
    # accumulate=1 over two calls against the accumulate path of the MSE loss
    eps1, _, _ = fixed(5, loss='mse')
    eps2, _, g_acc = fixed(6, loss='mse', accumulate=True)
    _vjp(eng, flat, mse_seed(eps1), seed=5)
    g, _, _ = _vjp(eng, flat, mse_seed(eps2), seed=6, accumulate=True)
    assert _bits_equal(g, g_acc)


# ---- 2./3. parity with the fp64 reference ---------------------------------------------------------------------------------------
def _parity_setup(dtype):
    S, B = 64, 2
    model = P.XUNet(**SMALL, dtype=dtype)
    rcfg = to_ref_cfg(model.config)
    ref_params = R.init_params(rcfg, S, seed=7, zero_init=False, bias_std=0.1)
    eng = model.engine(B, S, True)
    flat = model.flat_from_tree(ref_params, S, B)
    batch, _ = R.synthetic_batch(B, S, seed=1234)
    cond = np.array([1.0, 0.0], np.float32)
    eng.load_inputs(np_batch(batch), cond_mask=cond)
    d_eps = _d_eps(B, S, 9)
    g, dx, dz = _vjp(eng, flat, d_eps, train=False)
    gflat = {k: v.double().cpu() for k, v in R.flatten(model.tree_from_flat(g, S, B)).items()}
    args = (ref_params, batch, torch.from_numpy(cond).double(), d_eps.double().cpu(), rcfg)
    return gflat, dx.double().cpu(), dz.double().cpu(), args


def test_fp32_gradients_match_the_reference():
    gflat, dx, dz, args = _parity_setup('fp32')
    _, gref, dx_ref, dz_ref = vjp_ref.vjp(*args)
    total_ref = math.sqrt(sum(float((x ** 2).sum()) for x in gref.values()))
    floor = 1e-3 * total_ref / math.sqrt(len(gref))               # the per-leaf floor of the Frobenius / MSE parity tests
    bad = {}
    for key, gr in gref.items():
        rel = float(torch.linalg.norm((gflat[key] - gr).reshape(-1))) / (float(torch.linalg.norm(gr.reshape(-1))) + floor)
        if rel > 2e-3:
            bad[key] = rel
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]
    assert rel_l2(dx, dx_ref) < 2e-3 and rel_l2(dz, dz_ref) < 2e-3, (rel_l2(dx, dx_ref), rel_l2(dz, dz_ref))


def test_bf16_input_gradients_sit_on_the_bf16_noise_floor():
    """dx and dz held to the bar of the bf16 gradient-leaf tests: the engine's distance to the exact fp64 reference is below 3x
    the rounding-aware reference's own distance to it (floored by the median leaf floor)."""
    gflat, dx, dz, args = _parity_setup('bf16')
    _, g0, dx0, dz0 = vjp_ref.vjp(*args)
    _, g1, dx1, dz1 = vjp_ref.vjp(*args, bf16_inputs_ste=True)
    total = math.sqrt(sum(float((g.double() ** 2).sum()) for g in g0.values()))
    floor_abs = 1e-3 * total / math.sqrt(len(g0))
    leaf = lambda a, b, fa=floor_abs: float(torch.linalg.norm((a - b).reshape(-1))) / (float(torch.linalg.norm(b.reshape(-1))) + fa)
    med = float(np.median([leaf(g1[k], g0[k]) for k in g0]))
    ratios = {}
    for name, eng_v, emu_v, ref_v in (('dx', dx, dx1, dx0), ('dz', dz, dz1, dz0)):
        ratios[name] = leaf(eng_v, ref_v, 0.0) / max(leaf(emu_v, ref_v, 0.0), med)
    print(f'bf16 input gradients: engine/floor ratios {ratios}, median leaf floor {med:.3e}')
    assert max(ratios.values()) < 3.0, ratios


# ---- 4. the input-gradient kernel alone ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
@pytest.mark.parametrize('cfgd', [TINY, WIDE], ids=['ch32', 'ch256'])
@pytest.mark.parametrize('S', [16, 32])
def test_input_gradient_kernel_matches_fp64_conv_transpose(dtype, cfgd, S):
    B = 2
    model, flat, eng, _, _ = _setup(cfgd, dtype, B, S)
    _, dx, dz = _vjp(eng, flat, _d_eps(B, S, 13), train=False)
    dy = eng.read_tap('Conv_0', grad=True).double().cpu()                         # (2B,S,S,ch), the values the kernel read
    shape, off = eng.spec['Conv_0/kernel']
    w = flat[off:off + int(np.prod(shape))].view(shape)[0].double().cpu()          # (3,3,3,ch)
    want = torch.nn.grad.conv2d_input((2 * B, 3, S, S), w.permute(3, 2, 0, 1), dy.permute(0, 3, 1, 2), padding=1)
    want = want.permute(0, 2, 3, 1).reshape(B, 2, S, S, 3)
    for got, ref in ((dx.double().cpu(), want[:, 0]), (dz.double().cpu(), want[:, 1])):
        assert rel_l2(got, ref) < 1e-5
        border = torch.ones(S, S, dtype=torch.bool)
        border[1:-1, 1:-1] = False
        assert rel_l2(got[:, border], ref[:, border]) < 1e-5


# ---- 5. finite differences on the engine ----------------------------------------------------------------------------------------
def test_input_gradients_match_finite_differences_of_the_engine():
    # h = 2e-3 along a unit direction: the oracle evaluated in fp32 at this step lands within 2.3e-3 of the exact derivative
    # (seeds 3-6); 4e-3 already leaves 8e-3 of curvature error
    S, B, h = 16, 2, 2e-3
    model, flat, eng, batch, _ = _setup(TINY, 'fp32', B, S)
    nb = np_batch(batch)
    cond = np.array([1.0, 0.0], np.float32)
    d_eps = _d_eps(B, S, 17)
    _, dx, dz = _vjp(eng, flat, d_eps, train=False)
    rng = np.random.RandomState(19)
    for key, grad in (('x', dx), ('z', dz)):
        # a unit direction, so the step h*v has norm h (a step of 1e-2 per element leaves a 10-30 % curvature error), tilted
        # toward the computed gradient: along a purely random direction <grad, v> is ~|grad|/40 and drowns in the fp32 noise of
        # the forwards (1-2 %, measured with the oracle in fp32), while an error in the gradient still shows up as fd != <grad, v>
        g = grad.double().cpu().numpy()
        r = rng.randn(B, S, S, 3)
        v = r / np.linalg.norm(r) + g / np.linalg.norm(g)
        v /= np.linalg.norm(v)

        def f(sign):
            eng.load_inputs(dict(nb, **{key: nb[key] + sign * h * v}), cond_mask=cond)
            return float((eng.forward(flat, train=False).double() * d_eps.double()).sum())

        fd = (f(1) - f(-1)) / (2 * h)
        an = float((grad.double().cpu() * torch.from_numpy(v)).sum())
        assert abs(fd - an) <= 1e-2 * abs(an), (key, fd, an)
        eng.load_inputs(nb, cond_mask=cond)


# ---- 6. determinism and graph replay -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_repeats_bit_for_bit_and_graph_replay_gives_the_eager_bits(dtype):
    S, B = 16, 3
    model, flat, eng, _, _ = _setup(dict(TINY, dropout=0.1), dtype, B, S)
    d_eps = _d_eps(B, S, 23)
    a, b = _vjp(eng, flat, d_eps), _vjp(eng, flat, d_eps)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert bool((a[1] != 0).any()) and bool((a[2] != 0).any())
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        eng.forward(flat, train=True, seed=5)                       # warm-up on the capture stream, as TrainStep does
        eng.backward_vjp(flat, d_eps, dx=True, dz=True)
        stream.synchronize()
        with torch.cuda.graph(graph, stream=stream):
            eng.forward(flat, train=True, seed=5)
            eng.backward_vjp(flat, d_eps, dx=True, dz=True)
    torch.cuda.synchronize()
    eng.grads.zero_(); eng.dx.zero_(); eng.dz.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eng.grads, a[0]) and torch.equal(eng.dx, a[1]) and torch.equal(eng.dz, a[2])


# ---- 7. the gradient-bucket hook ----------------------------------------------------------------------------------------------
def test_bucket_hook_sees_the_ranges_of_the_mse_backward():
    S, B = 16, 2
    model, flat, eng, _, _ = _setup(TINY, 'bf16', B, S)
    seen = []
    n = eng.set_bucket_callback(lambda off, cnt: seen.append((off, cnt)), min_bucket_bytes=4096)
    try:
        eng.forward(flat, train=True, seed=1)
        eng.backward(flat, loss='mse')
        mse_ranges, seen[:] = list(seen), []
        _vjp(eng, flat, _d_eps(B, S, 29))
        vjp_ranges = list(seen)
    finally:
        eng.set_bucket_callback(None)
    assert len(mse_ranges) == n >= 2 and vjp_ranges == mse_ranges


# ---- 8. the Python surface ---------------------------------------------------------------------------------------------------
def test_vjp_fn_refuses_a_stale_forward_and_a_bad_seed():
    S, B = 16, 2
    model, flat, eng, batch, _ = _setup(TINY, 'bf16', B, S)
    nb = np_batch(batch)
    cond = np.array([1.0, 0.0], np.float32)
    eps, vjp_fn = model.vjp({'params': model.tree_from_flat(flat, S, B)}, nb, cond_mask=cond, train=False)
    d = _d_eps(B, S, 31)
    t1, in1 = vjp_fn(d)
    t2, in2 = vjp_fn(d)                                               # may be called again: same bits, independent copies
    assert torch.equal(t1.flat, t2.flat) and torch.equal(in1['x'], in2['x']) and torch.equal(in1['z'], in2['z'])
    assert t1.flat.data_ptr() != eng.grads.data_ptr() and in1['x'].data_ptr() != eng.dx.data_ptr()
    for bad in (d.double(), d.cpu(), d[:1], d.transpose(1, 2)):
        with pytest.raises(ValueError):
            vjp_fn(bad)
    eng.forward(flat, train=False)
    with pytest.raises(RuntimeError):
        vjp_fn(d)


def test_autograd_backward_equals_vjp_fn_bit_for_bit():
    S, B = 16, 2
    model, flat0, eng, batch, noise = _setup(dict(TINY, dropout=0.1), 'bf16', B, S)
    cond = np.array([1.0, 0.0], np.float32)
    nb = np_batch(batch)
    logsnr = torch.from_numpy(nb['logsnr']).float().cuda()
    alpha = torch.sigmoid(logsnr).sqrt().view(B, 1, 1, 1)
    sigma = torch.sigmoid(-logsnr).sqrt().view(B, 1, 1, 1)
    z_in = torch.from_numpy(nb['z']).float().cuda()
    noise_t = torch.from_numpy(noise).cuda()

    def v_loss(eps):
        """v-prediction target: v = alpha * eps - sigma * x0, with x0 recovered from z (a constant here)."""
        x0 = (z_in - sigma * noise_t) / alpha
        x0_hat = (z_in - sigma * eps) / alpha
        return ((alpha * eps - sigma * x0_hat) - (alpha * noise_t - sigma * x0)).pow(2).mean()

    flat = flat0.detach().clone().requires_grad_(True)
    x = torch.from_numpy(nb['x']).float().cuda().requires_grad_(True)
    z = z_in.clone().requires_grad_(True)
    eps = model.apply_autograd(flat, dict(nb, x=x, z=z), cond_mask=cond, train=True, rngs=7)
    assert eps.grad_fn is not None
    v_loss(eps).backward()

    eps2, vjp_fn = model.vjp({'params': model.tree_from_flat(flat0, S, B)}, nb, cond_mask=cond, train=True, rngs=7)
    assert torch.equal(eps.detach(), eps2)
    e = eps2.clone().requires_grad_(True)
    d_eps, = torch.autograd.grad(v_loss(e), e)
    tree, inputs = vjp_fn(d_eps.contiguous())
    assert torch.equal(flat.grad, tree.flat)
    assert torch.equal(x.grad, inputs['x']) and torch.equal(z.grad, inputs['z'])
    assert bool((x.grad != 0).any()) and bool((z.grad != 0).any())

    # an input that does not require grad gets none
    x2 = x.detach().clone()
    z.grad = None
    v_loss(model.apply_autograd(flat, dict(nb, x=x2, z=z), cond_mask=cond, train=False)).backward()
    assert x2.grad is None and z.grad is not None and bool((z.grad != 0).any())
    # a forward in between is refused
    eps = model.apply_autograd(flat, dict(nb, x=x, z=z), cond_mask=cond, train=False)
    eng.forward(flat0, train=False)
    with pytest.raises(RuntimeError):
        v_loss(eps).backward()
