"""GPU parity of the whole hot path through the reference-shaped API (XUNet.init/apply, apply_model, update_model,
Sampler) against the CPU oracle: fp32 verify mode to <=1e-3 relative (north_star), bf16 mode with the oracle fed the
same weights; per-block activation taps; all parameter gradients; Adam; sampler; metamorphic properties; golden vectors."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from tests.util import rel_l2, to_ref_cfg, np_batch, keep_mask
import novel_view_synthesis_3d_b200 as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')

TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)
TINY_POS = dict(TINY, use_pos_emb=True, use_ref_pose_emb=True)
SMALL = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4, dropout=0.1)
FOUR = dict(ch=64, ch_mult=(1, 2, 2, 4), emb_ch=128, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=8, dropout=0.0)   # full-3DiM topology, narrow
THREE = dict(ch=32, ch_mult=(1, 2, 2), emb_ch=64, num_res_blocks=1, attn_resolutions=(8,), attn_heads=1, dropout=0.0)

FWD_TOL = {'fp32': 1e-3, 'bf16': 4e-2}      # relative L2 on eps_hat (north_star: <=1e-3 in fp32; bf16: ~1e-2 expected from 2^-9 activation rounding)


def _setup(cfgd, S, B, dtype, seed=1234, params=None):
    """params: 'formula' (sinusoid leaves, badly conditioned: amplifies rounding ~100x -- a hard fp32 test) or 'random'
    (lecun-normal kernels incl. the zero-init ones, randomised biases: what a bf16 run can be held to)."""
    model = P.XUNet(**cfgd, dtype=dtype)
    rcfg = to_ref_cfg(model.config)
    params = params or ('formula' if dtype == 'fp32' else 'random')
    ref_params = R.formula_params(rcfg, S) if params == 'formula' else R.init_params(rcfg, S, seed=7, zero_init=False, bias_std=0.1)
    flat = model.flat_from_tree(ref_params, S, B)
    tree = model.tree_from_flat(flat, S, B)
    batch, noise = R.synthetic_batch(B, S, seed=seed)
    return model, rcfg, ref_params, tree, batch, noise


ODD = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(12,), attn_heads=2, dropout=0.0)   # S=24: no tile fits -> SIMT fallbacks


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
@pytest.mark.parametrize('cfgd,S,B', [(TINY, 16, 2), (TINY_POS, 16, 2), (THREE, 32, 1), (SMALL, 64, 2), (FOUR, 64, 1), (ODD, 24, 3)])
def test_forward_matches_oracle(cfgd, S, B, dtype):
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, dtype)
    cond = torch.tensor(([1.0, 0.0] * B)[:B], dtype=torch.float64)   # ragged conditioning: some samples unconditioned
    taps = {}
    ref = R.xunet_forward(ref_params, batch, cond, rcfg, train=False, taps=taps)
    eps = model.apply({'params': tree}, np_batch(batch), cond_mask=cond.numpy(), train=False)
    assert eps.shape == (B, S, S, 3) and eps.dtype == torch.float32
    eng = model.engine(B, S, False)
    errs = {}
    for name in eng.taps():
        if name in taps:
            t = taps[name]
            errs[name] = rel_l2(eng.read_tap(name), t.reshape(-1, *t.shape[-3:]) if t.dim() == 5 else t.reshape(B, 1, 1, -1))
    worst = max(errs.values())
    assert worst < FWD_TOL[dtype] * 2, sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    assert rel_l2(eps, ref) < FWD_TOL[dtype], errs


@pytest.mark.parametrize('name', ['tiny16_b2', 'small64_b2'])
def test_forward_matches_golden_fixture(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_golden', os.path.join(GOLD, 'make_golden.py'))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    rcfg, S, B = mg.CASES[name]
    gold = np.load(os.path.join(GOLD, name + '.npz'))
    cfgd = dict(ch=rcfg.ch, ch_mult=rcfg.ch_mult, emb_ch=rcfg.emb_ch, num_res_blocks=rcfg.num_res_blocks,
                attn_resolutions=rcfg.attn_resolutions, attn_heads=rcfg.attn_heads, dropout=rcfg.dropout,
                use_pos_emb=rcfg.use_pos_emb, use_ref_pose_emb=rcfg.use_ref_pose_emb)
    model, _, _, tree, batch, _ = _setup(cfgd, S, B, 'fp32')
    eps = model.apply({'params': tree}, np_batch(batch), cond_mask=gold['cond_mask'], train=False)
    assert rel_l2(eps, gold['eps']) < 1e-3


GRAD_CASES = [
    # cfg, S, B, dropout, params, dtype, per-leaf tol
    (TINY_POS, 16, 2, 0.0, 'formula', 'fp32', 5e-3), (TINY_POS, 16, 2, 0.0, 'random', 'bf16', 2e-1),
    (THREE, 32, 1, 0.0, 'random', 'fp32', 2e-3), (THREE, 32, 1, 0.0, 'random', 'bf16', 2e-1),
    (SMALL, 64, 2, 0.1, 'random', 'fp32', 2e-3), (SMALL, 64, 2, 0.1, 'random', 'bf16', 2e-1),
    (FOUR, 64, 1, 0.0, 'random', 'bf16', 2e-1),
]


@pytest.mark.parametrize('cfgd,S,B,drop,pkind,dtype,gtol', GRAD_CASES)
def test_train_step_gradients_match_oracle(cfgd, S, B, drop, pkind, dtype, gtol):
    cfgd = dict(cfgd, dropout=drop)
    model, rcfg, ref_params, tree, batch, noise = _setup(cfgd, S, B, dtype, params=pkind)
    cond = np.array(([1.0, 0.0] * B)[:B])
    state = P.create_train_state(0, 1, 1e-4, B, S, model=model)
    state.params.flat.copy_(tree.flat)
    nb = np_batch(batch)
    seed = state.step + 1
    mask_fn = (lambda idx, shape: torch.from_numpy(keep_mask(seed, idx, shape, drop))) if drop > 0 else None
    loss_ref, grads_ref, _ = R.loss_and_grads(ref_params, batch, noise, torch.from_numpy(cond), rcfg, train=True,
                                              drop_mask_fn=mask_fn)
    loss, grads = P.apply_model(state, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'],
                                noise.numpy(), cond_mask=cond)
    ltol = 2e-4 if dtype == 'fp32' else 2e-2
    assert abs(float(loss) - float(loss_ref)) / float(loss_ref) < ltol
    gflat = R.flatten(grads)
    total_ref = math.sqrt(sum(float((g ** 2).sum()) for g in grads_ref.values()))
    bad, worst = {}, (0.0, '')
    for k, gr in grads_ref.items():
        gg = gflat[k].double().cpu()
        err = float(torch.linalg.norm((gg - gr).reshape(-1)))
        # per-leaf relative error, floored so leaves with negligible gradient do not dominate
        rel = err / (float(torch.linalg.norm(gr.reshape(-1))) + 1e-3 * total_ref / math.sqrt(len(grads_ref)))
        worst = max(worst, (rel, k))
        # bf16 activation gradients: bias / GroupNorm leaves are plain sums of ~1e5 rounded terms with heavy
        # cancellation, so only the GEMM-shaped (kernel) leaves are held to the per-leaf bound there
        strict = dtype == 'fp32' or k.endswith('kernel')
        if rel > (gtol if strict else 1.0):
            bad[k] = rel
    all_g = torch.cat([gflat[k].double().cpu().reshape(-1) for k in grads_ref])
    all_r = torch.cat([g.reshape(-1) for g in grads_ref.values()])
    glob = rel_l2(all_g, all_r)
    print(f'grad parity [{dtype},{pkind}]: global rel-L2 {glob:.3e}, worst leaf {worst[1]} {worst[0]:.3e}')
    assert not bad, (glob, sorted(bad.items(), key=lambda kv: -kv[1])[:8])
    assert glob < gtol / 2, glob

    # update_model == optax.adam on every leaf
    new_state = P.update_model(state, grads)
    assert new_state.step == 1
    flat_ref = R.flatten(ref_params)
    for k in list(flat_ref)[:: max(1, len(flat_ref) // 12)]:
        p_new, _, _ = R.adam_update(flat_ref[k], grads_ref[k], torch.zeros_like(grads_ref[k]), torch.zeros_like(grads_ref[k]), 1)
        got = R.flatten(new_state.params)[k].double().cpu()
        # Adam's first step is -lr*sign(g): only compare where the oracle gradient is not tiny
        sel = grads_ref[k].abs() > 1e-4 * grads_ref[k].abs().max() + 1e-12
        if not bool(sel.any()):
            continue
        assert float((got - p_new)[sel].abs().max()) < (2e-6 if dtype == 'fp32' else 2.1e-4), k


def test_zero_init_cond_mask_and_frame_swap_properties():
    model = P.XUNet(**TINY, dtype='fp32')
    S, B = 16, 2
    batch, _ = R.synthetic_batch(B, S, seed=5)
    nb = np_batch(batch)
    v0 = model.init({'params': 3, 'dropout': 4}, nb, cond_mask=np.zeros(B), train=True)
    assert float(model.apply(v0, nb, cond_mask=np.ones(B), train=False).abs().max()) == 0.0     # SURVEY F9
    v = model.init({'params': 3, 'dropout': 4}, nb, cond_mask=np.zeros(B), train=True, zero_init=False)
    o, _ = R.synthetic_batch(B, S, seed=99)
    nb2 = dict(nb, **{k: o[k].numpy() for k in ('R1', 't1', 'R2', 't2')})
    a = model.apply(v, nb, cond_mask=np.zeros(B), train=False)
    b = model.apply(v, nb2, cond_mask=np.zeros(B), train=False)
    assert rel_l2(a, b) < 1e-5      # pose-invariant when unconditioned (fp32 atomics make runs differ in the last bits)
    assert rel_l2(model.apply(v, nb, cond_mask=np.ones(B), train=False), model.apply(v, nb2, cond_mask=np.ones(B), train=False)) > 1e-4
    # frame swap: target-frame output of (x,z,cam1,cam2) == source-frame output of (z,x,cam2,cam1)
    eng = model.engine(B, S, False)
    model.apply(v, nb, cond_mask=np.ones(B), train=False)
    both = eng.read_tap('out_both_frames').reshape(B, 2, S, S, 3)
    sw = dict(nb, x=nb['z'], z=nb['x'], R1=nb['R2'], t1=nb['t2'], R2=nb['R1'], t2=nb['t1'])
    model.apply(v, sw, cond_mask=np.ones(B), train=False)
    both_sw = eng.read_tap('out_both_frames').reshape(B, 2, S, S, 3)
    assert rel_l2(both[:, 1], both_sw[:, 0]) < 1e-4 and rel_l2(both[:, 0], both_sw[:, 1]) < 1e-4
    with pytest.raises(AssertionError):
        model.apply(v, nb, cond_mask=np.ones(B + 1), train=False)                               # model/xunet.py:176


def test_dropout_train_mode_is_seeded_and_unbiased():
    model = P.XUNet(**dict(TINY, dropout=0.3), dtype='fp32')
    S, B = 16, 2
    batch, _ = R.synthetic_batch(B, S, seed=5)
    nb = np_batch(batch)
    v = model.init({'params': 1}, nb, cond_mask=np.zeros(B), zero_init=False)
    ones = np.ones(B)
    a = model.apply(v, nb, cond_mask=ones, train=True, rngs={'dropout': 7})
    b = model.apply(v, nb, cond_mask=ones, train=True, rngs={'dropout': 7})
    c = model.apply(v, nb, cond_mask=ones, train=True, rngs={'dropout': 8})
    e = model.apply(v, nb, cond_mask=ones, train=False)
    # GroupNorm statistics are accumulated with fp32 atomics -> last-bit run-to-run differences, not bit equality
    assert rel_l2(a, b) < 1e-5 and rel_l2(a, c) > 1e-2 and rel_l2(a, e) > 1e-2


def test_train_step_class_matches_apply_update_and_learns():
    S, B = 16, 4
    batch, noise = R.synthetic_batch(B, S, seed=21)
    nb = np_batch(batch)
    cond = np.ones(B, dtype=np.float32)
    losses = {}
    for use_graph in (False, True):
        model = P.XUNet(**TINY, dtype='fp32')
        st = P.create_train_state(0, 1, 1e-3, B, S, model=model, zero_init=False)
        step = P.TrainStep(st, use_graph=use_graph)
        losses[use_graph] = [float(step(nb, noise.numpy(), cond_mask=cond)) for _ in range(6)]
        assert st.step == 6
    assert np.allclose(losses[False], losses[True], rtol=3e-3)   # Adam's sign-like early steps amplify last-bit differences
    assert losses[True][-1] < losses[True][0]                    # same batch every step -> the loss must go down
    # reference-shaped two-call API gives the same first loss
    model = P.XUNet(**TINY, dtype='fp32')
    st = P.create_train_state(0, 1, 1e-3, B, S, model=model, zero_init=False)
    l0, g = P.apply_model(st, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'], noise.numpy(), cond_mask=cond)
    assert abs(float(l0) - losses[False][0]) / losses[False][0] < 1e-4


def test_sampler_matches_oracle_loop():
    """Last 3 steps of the 1000-step reference sampler (sampling.py:128-151) with shared noise."""
    cfgd, S, B = TINY, 16, 1
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, 'fp32')
    nb = np_batch(batch)
    g = torch.Generator().manual_seed(9)
    steps = 4
    z0 = torch.randn(B, S, S, 3, generator=g, dtype=torch.float64)
    noises = [torch.randn(B, S, S, 3, generator=g, dtype=torch.float64) for _ in range(steps)]
    samp = P.Sampler(model, tree, B, S, steps=1000, w=3.0, use_graph=True)
    # run only the last `steps` timesteps: emulate by truncating the schedule
    samp.sched.timesteps = samp.sched.timesteps[:steps]
    for k in ('sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod', 'posterior_mean_coef1', 'posterior_mean_coef2',
              'posterior_log_variance_clipped'):
        setattr(samp.sched, k, getattr(samp.sched, k)[:steps])
    out = samp.sample(nb, z_init=z0.numpy(), noises=[n.numpy() for n in noises])
    tab = R.schedule_tables()
    z, logsnr = z0, -20.0
    for i, t in enumerate(range(steps - 1, -1, -1)):
        b = dict(batch, z=z, logsnr=torch.full((B,), logsnr, dtype=torch.float64))
        ec = R.xunet_forward(ref_params, b, torch.ones(B), rcfg)
        eu = R.xunet_forward(ref_params, b, torch.zeros(B), rcfg)
        z, logsnr = R.sampler_step(ec, eu, z, t, noises[i], tab)
    assert rel_l2(out, z) < 2e-3


def _pool_from_batch(nb):
    """(views, poses, K, target_poses) of sample_views() from a data-loader style batch: source = frame 1, target = frame 2."""
    return (nb['x'][:, None], {'R': nb['R1'][:, None], 't': nb['t1'][:, None]}, nb['K'],
            {'R': nb['R2'][:, None], 't': nb['t2'][:, None]})


def test_stochastic_conditioning_reduces_to_the_k1_sampler():
    """SURVEY 8(f) row 4: with one source view and one target the multi-view loop IS the reference's k=1 sampler."""
    cfgd, S, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, 'fp32')
    nb = np_batch(batch)
    samp = P.Sampler(model, tree, B, S, steps=6, w=3.0)
    a = samp.sample(nb, seed=3)
    views, poses, K, tp = _pool_from_batch(nb)
    b, ch = samp.sample_views(views, poses, K, tp, seed=3, return_choices=True)
    assert ch.shape == (1, 6) and (ch == 0).all()
    # the same kernels on the same inputs (sample() reuses the first step's pose embeddings and weight shadows), but the fp64
    # GroupNorm sums are order-insensitive only with overwhelming probability, not by construction: compare with a tolerance
    assert rel_l2(b[:, 0], a) < 2e-3


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_graph_replay_and_eager_sampling_are_bit_identical(dtype):
    """use_graph=True replays the forward + table step + position increment that use_graph=False issues eagerly."""
    cfgd, S, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, dtype)
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {k: np.concatenate([tp[k], poses[k]], 1) for k in ('R', 't')}      # two targets: the second reuses the graph
    out = {}
    for use_graph in (True, False):
        samp = P.Sampler(model, tree, B, S, steps=6, w=3.0, use_graph=use_graph)
        out[use_graph] = (samp.sample(nb, seed=3), samp.sample_views(views, poses, K, tp, seed=3))
    assert torch.equal(out[True][0], out[False][0])
    assert torch.equal(out[True][1], out[False][1])


def test_stochastic_conditioning_matches_oracle_loop():
    """Two source views, two targets, pool growing with the generated view: every step's conditioning view is the one the
    sampler drew; the oracle replays the same draws (sampling.py:128-151 per step)."""
    cfgd, S, B = TINY, 16, 1
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, 'fp32')
    b2, _ = R.synthetic_batch(B, S, seed=77)
    nb, nb2 = np_batch(batch), np_batch(b2)
    steps, m = 3, 2
    views = np.stack([nb['x'], nb2['x']], 1)
    poses = {'R': np.stack([nb['R1'], nb2['R1']], 1), 't': np.stack([nb['t1'], nb2['t1']], 1)}
    tp = {'R': np.stack([nb['R2'], nb2['R2']], 1), 't': np.stack([nb['t2'], nb2['t2']], 1)}
    g = torch.Generator().manual_seed(11)
    z0 = torch.randn(m, B, S, S, 3, generator=g, dtype=torch.float64)
    noises = torch.randn(m, steps, B, S, S, 3, generator=g, dtype=torch.float64)
    samp = P.Sampler(model, tree, B, S, steps=1000, w=3.0, use_graph=True)
    samp.sched.timesteps = samp.sched.timesteps[:steps]
    for k in ('sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod', 'posterior_mean_coef1', 'posterior_mean_coef2',
              'posterior_log_variance_clipped'):
        setattr(samp.sched, k, getattr(samp.sched, k)[:steps])
    out, ch = samp.sample_views(views, poses, nb['K'], tp, seed=5, return_choices=True, z_init=z0.numpy(), noises=noises.numpy())
    assert ch.shape == (m, steps) and ch[0].max() < 2 and ch[1].max() < 3
    tab = R.schedule_tables()
    t64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)
    pool = [(t64(views[:, i]), t64(poses['R'][:, i]), t64(poses['t'][:, i])) for i in range(2)]
    for j in range(m):
        z, logsnr = z0[j], -20.0
        for i, t in enumerate(range(steps - 1, -1, -1)):
            px, pR, pt = pool[ch[j, i]]
            b = dict(x=px, z=z, logsnr=torch.full((B,), logsnr, dtype=torch.float64), R1=pR, t1=pt,
                     R2=t64(tp['R'][:, j]), t2=t64(tp['t'][:, j]), K=t64(nb['K']))
            ec = R.xunet_forward(ref_params, b, torch.ones(B), rcfg)
            eu = R.xunet_forward(ref_params, b, torch.zeros(B), rcfg)
            z, logsnr = R.sampler_step(ec, eu, z, t, noises[j, i], tab)
        assert rel_l2(out[:, j], z) < 2e-3, j
        pool.append((z, t64(tp['R'][:, j]), t64(tp['t'][:, j])))


def test_flax_checkpoint_roundtrip_drives_the_gpu_path(tmp_path):
    """sampling.py:106-114: parameters restored from a (device-axis) Flax msgpack checkpoint run on the CUDA path."""
    from novel_view_synthesis_3d_b200 import checkpoint as ck
    model = P.XUNet(**TINY, dtype='fp32')
    S, B = 16, 2
    batch, _ = R.synthetic_batch(B, S, seed=5)
    nb = np_batch(batch)
    v = model.init({'params': 11}, nb, cond_mask=np.zeros(B), zero_init=False)
    ref = model.apply(v, nb, cond_mask=np.ones(B), train=False)
    ck.save_checkpoint(str(tmp_path), v['params'], step=0, prefix='model', add_device_axis=True)
    tree = ck.restore_checkpoint(str(tmp_path), prefix='model0')          # the prefix sampling.py:109 uses
    assert tree is not None
    out = model.apply({'params': tree}, nb, cond_mask=np.ones(B), train=False)
    assert rel_l2(out, ref) < 1e-5


def test_device_forward_diffusion_matches_data_loader_formulas():
    """dataset/data_loader.py:92-110 on the GPU: z = sqrt(abar_t) x0 + sqrt(1-abar_t) eps, logsnr cosine schedule, t in [0,1000)."""
    model = P.XUNet(**TINY, dtype='fp32')
    S, B = 16, 4
    eng = model.engine(B, S, True)
    fd = P.ForwardDiffusion(eng)
    g = torch.Generator().manual_seed(3)
    x0 = torch.rand(B, S, S, 3, generator=g) * 2 - 1
    noise = torch.randn(B, S, S, 3, generator=g)
    t = np.array([0, 1, 500, 999], dtype=np.int32)
    fd.sample(x0, seed=5, t=t, noise=noise)
    torch.cuda.synchronize()
    tab = R.schedule_tables()
    z_ref = tab['sqrt_alphas_cumprod'][t][:, None, None, None] * x0.double().numpy() + \
        tab['sqrt_one_minus_alphas_cumprod'][t][:, None, None, None] * noise.double().numpy()
    assert rel_l2(eng.inp['z'], z_ref) < 1e-6
    assert np.allclose(eng.inp['logsnr'].cpu().numpy(), R.logsnr_schedule_cosine(t / 1000.0), rtol=1e-5, atol=1e-5)
    # device-drawn t / noise / cond_mask: ranges and moments
    eng2 = model.engine(64, S, True)
    fd2 = P.ForwardDiffusion(eng2)
    fd2.sample(torch.zeros(64, S, S, 3), seed=11)
    torch.cuda.synchronize()
    tt = fd2.t.cpu().numpy()
    assert tt.min() >= 0 and tt.max() < 1000 and len(np.unique(tt)) > 32
    nz = eng2.inp['noise']
    assert abs(float(nz.mean())) < 2e-2 and abs(float(nz.std()) - 1) < 2e-2
    # x0 = 0 -> z = sqrt(1-abar_t) * noise exactly
    s1 = torch.as_tensor(tab['sqrt_one_minus_alphas_cumprod'][tt], dtype=torch.float32).cuda()[:, None, None, None]
    assert rel_l2(eng2.inp['z'], s1 * nz) < 1e-6
    cm = eng2.inp['cond_mask'].cpu().numpy()
    assert set(np.unique(cm)) <= {0.0, 1.0} and 0.6 < cm.mean() <= 1.0
    fd2.sample(torch.zeros(64, S, S, 3), seed=12)
    torch.cuda.synchronize()
    assert not np.array_equal(fd2.t.cpu().numpy(), tt)


def test_end_to_end_srn_tree_train_checkpoint_sample(tmp_path):
    """The reference's two scripts end to end on a synthetic SRN tree: reader -> device forward diffusion -> fused train step
    -> Flax-format checkpoint -> restore -> CFG sampler -> PNG."""
    cv2 = pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    from novel_view_synthesis_3d_b200.srn_data import SRNScenes
    root = str(tmp_path / 'cars')
    _make_tree(root, n_inst=2, n_views=4, H=32, W=32)
    S, B = 16, 2
    ds = SRNScenes(root, img_sidelength=S, seed=0)
    model = P.XUNet(**TINY, dtype='bf16')
    state = P.create_train_state(0, 1, 1e-3, B, S, model=model, zero_init=False)
    step = P.TrainStep(state)
    fd = P.ForwardDiffusion(step.eng)
    stream = ds.batches(B)
    losses = []
    for it in range(4):
        b = next(stream)
        fd.sample(b['target'], seed=it)
        dev = step.eng.inp
        batch = {k: b[k] for k in ('x', 'R1', 't1', 'R2', 't2', 'K')}
        batch.update(z=dev['z'], logsnr=dev['logsnr'])
        losses.append(float(step(batch, dev['noise'], cond_mask=dev['cond_mask'])))
    assert all(np.isfinite(losses)) and state.step == 4
    P.checkpoint.save_checkpoint(str(tmp_path / 'ck'), state.params, step=0, add_device_axis=True)
    params = P.checkpoint.restore_checkpoint(str(tmp_path / 'ck'), prefix='model0')
    b = next(stream)
    z = P.Sampler(model, params, B, S, steps=8, w=3.0).sample(b, seed=1)
    assert z.shape == (B, S, S, 3) and bool(torch.isfinite(z).all())
    out = str(tmp_path / 'view.png')
    P.sampling.save_view(out, z[0].cpu().numpy())
    assert cv2.imread(out).shape == (S, S, 3)
