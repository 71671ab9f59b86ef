"""xunet_image_metrics (MSE / PSNR / SSIM on the device) against the float64 reference of tests/ssim_ref.py, its determinism,
graph capture and argument checks, and examples/eval_srn.py end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from tests import ssim_ref as M

pytestmark = pytest.mark.gpu


def _bits(m):
    return {k: v.cpu().numpy().view(np.uint32).copy() for k, v in m.items()}


def _mixed_batch(B, S):
    """B images of alternating kinds (so every position holds a different kind of pair)."""
    pairs = [M.make_pair(M.PAIR_KINDS[i % len(M.PAIR_KINDS)], 1, S, seed=100 + i) for i in range(B)]
    return np.concatenate([p for p, _ in pairs]), np.concatenate([t for _, t in pairs])


# ---- 1. against the float64 reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 3, 8])
@pytest.mark.parametrize('S', [11, 16, 64, 128, 256])
@pytest.mark.parametrize('kind', M.PAIR_KINDS)
def test_kernel_matches_reference(kind, S, B):
    p, t = M.make_pair(kind, B, S, seed=S * 10 + B)
    got = {k: v.cpu().numpy().astype(np.float64) for k, v in P.image_metrics(p, t).items()}
    assert all(v.shape == (B,) for v in got.values())
    mse, psnr = M.mse_psnr(p, t)
    ssim = M.ssim(p, t)
    if kind == 'identical':
        assert np.all(got['mse'] == 0) and np.all(np.isposinf(got['psnr']))
        assert np.all(np.abs(got['ssim'] - 1.0) <= 1e-6), got['ssim']
        return
    assert np.all(np.abs(got['ssim'] - ssim) <= 1e-5), (got['ssim'], ssim)
    assert np.all(np.abs(got['psnr'] - psnr) <= 1e-4), (got['psnr'], psnr)
    assert np.all(np.abs(got['mse'] - mse) <= 1e-6 * mse), (got['mse'], mse)


def test_known_answers_on_the_device():
    S = 32
    a, b = np.float32(0.5), np.float32(-0.25)
    m = P.image_metrics(np.full((1, S, S, 3), a), np.full((1, S, S, 3), b))
    ua, ub = (np.float64(a) + 1) / 2, (np.float64(b) + 1) / 2
    assert abs(m['ssim'].item() - (2 * ua * ub + M.C1) / (ua * ua + ub * ub + M.C1)) <= 1e-6
    rng = np.random.RandomState(3)
    t = rng.uniform(-0.9, 0.7, (2, S, S, 3)).astype(np.float32)
    p = t + np.float32(0.2)
    assert np.allclose(P.image_metrics(p, t)['psnr'].cpu().numpy(), M.mse_psnr(p, t)[1], rtol=0, atol=1e-4)
    assert np.allclose(P.image_metrics(p, t)['psnr'].cpu().numpy(), 20.0, rtol=0, atol=1e-3)
    wide = (1.5 * rng.uniform(-1, 1, (2, S, S, 3))).astype(np.float32)
    a, b = _bits(P.image_metrics(wide, t)), _bits(P.image_metrics(np.clip(wide, -1, 1), t))
    assert all(np.array_equal(a[k], b[k]) for k in a)               # inputs outside [-1, 1] score as their clamped values


# ---- 2. determinism ---------------------------------------------------------------------------------------------------------
def test_repeat_calls_are_bit_identical():
    p, t = (torch.as_tensor(x).cuda() for x in _mixed_batch(8, 128))
    a, b = _bits(P.image_metrics(p, t)), _bits(P.image_metrics(p, t))
    assert all(np.array_equal(a[k], b[k]) for k in a)


def test_an_image_scores_the_same_alone_and_anywhere_in_a_batch():
    p, t = _mixed_batch(8, 64)
    full = _bits(P.image_metrics(p, t))
    perm = np.random.RandomState(0).permutation(8)
    shuffled = _bits(P.image_metrics(p[perm], t[perm]))
    for i in range(8):
        alone = _bits(P.image_metrics(p[i:i + 1], t[i:i + 1]))
        j = int(np.nonzero(perm == i)[0][0])
        for k in full:
            assert full[k][i] == alone[k][0] == shuffled[k][j], (k, i)


# ---- 3. graph capture, input kinds ------------------------------------------------------------------------------------------
def test_graph_replay_equals_eager_on_new_contents():
    p0, t0 = M.make_pair('srn', 3, 64, seed=1)
    p1, t1 = M.make_pair('smooth', 3, 64, seed=2)
    p, t = torch.as_tensor(p0).cuda(), torch.as_tensor(t0).cuda()
    P.image_metrics(p, t)                       # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = P.image_metrics(p, t)
    p.copy_(torch.as_tensor(p1))
    t.copy_(torch.as_tensor(t1))
    g.replay()
    torch.cuda.synchronize()
    want = _bits(P.image_metrics(p1, t1))
    got = _bits(out)
    assert all(np.array_equal(got[k], want[k]) for k in want)


def test_numpy_and_device_inputs_agree():
    p, t = M.make_pair('noise', 3, 32, seed=4)
    a = _bits(P.image_metrics(p, t))
    b = _bits(P.image_metrics(torch.as_tensor(p).cuda(), torch.as_tensor(t).cuda()))
    c = _bits(P.image_metrics(torch.as_tensor(p.astype(np.float64)), t))     # a CPU float64 tensor is converted too
    assert all(np.array_equal(a[k], b[k]) and np.array_equal(a[k], c[k]) for k in a)


# ---- 4. errors --------------------------------------------------------------------------------------------------------------
def test_c_abi_rejects_bad_arguments(lib):
    x = torch.zeros(2, 16, 16, 3, device='cuda')
    out = torch.zeros(3, 2, device='cuda')
    o = [out[i].data_ptr() for i in range(3)]
    st = torch.cuda.current_stream().cuda_stream
    cases = {'S < 11': (x.data_ptr(), x.data_ptr(), 2, 10, *o), 'S > max': (x.data_ptr(), x.data_ptr(), 2, 257, *o),
             'B = 0': (x.data_ptr(), x.data_ptr(), 0, 16, *o), 'pred NULL': (None, x.data_ptr(), 2, 16, *o),
             'target NULL': (x.data_ptr(), None, 2, 16, *o), 'ssim NULL': (x.data_ptr(), x.data_ptr(), 2, 16, o[0], o[1], None)}
    for what, args in cases.items():
        assert lib.xunet_image_metrics(*args, st) != 0, what
        assert lib.xunet_last_error().decode().startswith('xunet_image_metrics'), what
    assert lib.xunet_image_metrics(x.data_ptr(), x.data_ptr(), 2, 16, *o, st) == 0


def test_python_rejects_bad_shapes():
    a = np.zeros((2, 16, 16, 3), np.float32)
    for bad in (np.zeros((2, 16, 16, 4), np.float32), np.zeros((2, 16, 8, 3), np.float32), np.zeros((16, 16, 3), np.float32)):
        with pytest.raises(ValueError):
            P.image_metrics(bad, bad)
    with pytest.raises(ValueError):
        P.image_metrics(a, np.zeros((3, 16, 16, 3), np.float32))
    with pytest.raises(ValueError):
        P.image_metrics(np.zeros((1, 8, 8, 3), np.float32), np.zeros((1, 8, 8, 3), np.float32))


# ---- 5. examples/eval_srn.py ------------------------------------------------------------------------------------------------
def test_eval_script_end_to_end(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    root, ck_dir = str(tmp_path / 'cars'), str(tmp_path / 'ck')
    _make_tree(root, n_inst=2, n_views=6, H=64, W=64)
    params = P.XUNet().init({'params': 3}, {'x': np.zeros((1, 64, 64, 3), np.float32)}, zero_init=False)['params']
    P.checkpoint.save_checkpoint(ck_dir, params, step=0, prefix='model', add_device_axis=True)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(out, *args):
        r = subprocess.run([sys.executable, os.path.join(repo, 'examples', 'eval_srn.py'), root, '--ckpt', ck_dir,
                            '--side', '64', '--steps', '4', '--out', out, *args], capture_output=True, text=True, timeout=600)
        return r

    for mode, vif in (('independent', '2'), ('stochastic', '2')):
        args = ('--source-view', '1', '--targets', '3', '--views-in-flight', vif, '--mode', mode, '--seed', '5')
        outs = [str(tmp_path / f'{mode}{k}') for k in range(2)]
        r = run(outs[0], *args, '--save-views')
        assert r.returncode == 0, r.stdout + r.stderr
        lines = [json.loads(s) for s in open(os.path.join(outs[0], 'metrics.jsonl'))]
        assert len(lines) == 2 * 3
        assert [(d['instance'], d['view']) for d in lines] == [(f'obj{i}', v) for i in range(2) for v in (0, 2, 4)], lines
        psnr, ssim = np.array([d['psnr'] for d in lines]), np.array([d['ssim'] for d in lines])
        assert np.all(np.isfinite(psnr)) and np.all(np.isfinite(ssim)) and np.all(np.abs(ssim) <= 1)
        summary = json.load(open(os.path.join(outs[0], 'summary.json')))
        assert json.loads(r.stdout.strip().splitlines()[-1]) == summary
        assert summary['n_views'] == 6 and summary['args']['mode'] == mode
        assert np.isclose(summary['mean_psnr'], psnr.mean(), rtol=1e-12) and np.isclose(summary['mean_ssim'], ssim.mean(), rtol=1e-12)
        assert len(os.listdir(os.path.join(outs[0], 'views'))) == 6
        r = run(outs[1], *args)
        assert r.returncode == 0, r.stdout + r.stderr
        assert open(os.path.join(outs[0], 'metrics.jsonl'), 'rb').read() == open(os.path.join(outs[1], 'metrics.jsonl'), 'rb').read()

    r = run(str(tmp_path / 'bad'), '--source-view', '6', '--targets', '2')
    assert r.returncode != 0 and 'obj0' in r.stderr and '--source-view 6' in r.stderr, r.stderr
