"""The benchmarked plans compute the same result however they are scheduled.

The per-launch tests (test_gpu_plan_launches.py, test_gpu_plan_ops.py) run each launch alone on one stream.  The engine runs
them differently: weight gradients and the FiLM branch on a side stream joined by events, every launch with programmatic
dependent launch (PDL), the step replayed from a CUDA graph, gradient buckets handed to an all-reduce hook mid-backward, and
grids, tile widths and split factors derived from the SM count.  Each child process below builds every plan of
launch_ref.PLANS in one such setting (the switches are read once per process) and records what the step computed:

  * the loss, eps_hat, every tap of the workspace (activations and gradients), the flat gradient and the Adam-updated
    parameters per leaf; on full128 also backward_vjp_inputs (dx, dz, the camera gradients) and a backward_accumulate pair;
    for the samplers three steps with static conditioning (z, eps_hat and the taps).
Large tensors are recorded as two 64-bit sums of their raw 32-bit words (plain and position-weighted): equal bytes give equal
sums, NaNs included, and one changed word changes both.

Schedule invariance: XUNET_NO_SIDE_STREAM=1 XUNET_NO_PDL=1 (fully serialised) is the reference.  The default (eager and
graph-replayed), XUNET_NO_PDL alone and XUNET_NO_SIDE_STREAM alone change only the order between kernels, never which kernel
runs, its grid or the fp64 scratch it folds into (one per stream), so every recorded tensor must carry the same bits.

Buckets: a hook installed with Engine.set_bucket_callback enqueues a copy of grads[off:off+n] on the backward's stream when
the engine hands the bucket out, as an all-reduce would read it; every copy must equal the final gradient.

SM count: with XUNET_SM_RESERVE the conv tile width (BN), persistent grid (ctas), CTAs per SM, pipeline depth, warpgroup
schedule and weight-gradient split-K factor change.  Every conv launch whose logged variant (XUNET_CONV_LOG) differs from the
unreserved one goes through the fp64 checks of test_gpu_plan_launches.test_conv_launch again in that child.  The whole step
is compared with the reference as well (see test_sm_reserve_step).
"""
import dataclasses
import gc
import math
import os
import re
import time

import numpy as np
import pytest
import torch

from tests import launch_ref as L

pytestmark = pytest.mark.gpu

REF = {'XUNET_NO_SIDE_STREAM': '1', 'XUNET_NO_PDL': '1'}
MODES = {'default': {}, 'no_pdl': {'XUNET_NO_PDL': '1'}, 'no_side_stream': {'XUNET_NO_SIDE_STREAM': '1'}}
SMALL_PLANS = ('small64', 'small128', 'small64_f32')
# SMs left free -> SMs used on a 132-SM H100: 114 (an H100 PCIe), 65, and 2 (small plans only, to bound the runtime)
RESERVES = {18: tuple(L.PLANS), 67: tuple(L.PLANS), 130: SMALL_PLANS}
# whose launches are re-checked against fp64 at each reserve: every plan at 65 SMs, the small plans at the others.  The fp64
# references of the full model's launches take about six minutes per reserve, so full64 and full128 launches that change
# variant only at 114 SMs are not re-checked; the 65-SM run covers the same kernels and split rules on both full plans.
RECHECK = {18: SMALL_PLANS, 67: tuple(L.PLANS), 130: SMALL_PLANS}
SWITCHES = ('XUNET_NO_SIDE_STREAM', 'XUNET_NO_PDL', 'XUNET_SM_RESERVE', 'XUNET_CONV_LOG')
FULL_LIMIT = 1 << 24        # tensors of up to this many bytes are recorded whole as well
VARIANT = ('BN', 'ctas', 'per_sm', 'stages', 'sched', 'ksplit')


# ======================================================================================================================
# child side
# ======================================================================================================================
def _fp(t):
    """(sum, position-weighted sum) of the raw bytes of t read as int32 words, in int64 arithmetic (wrapping)"""
    b = t.contiguous().view(torch.uint8).reshape(-1)
    if b.storage_offset() % 4:
        b = b.clone()
    if b.numel() % 4:
        b = torch.cat([b, b.new_zeros(4 - b.numel() % 4)])
    w = b.view(torch.int32).to(torch.int64)
    i = torch.arange(w.numel(), device=w.device, dtype=torch.int64)
    return int(w.sum()), int((w * (i * 0x9E3779B1 + 0x632BE5AB)).sum())


def _rec(t):
    """fingerprint of a tensor, and the tensor itself (on the host) when it is small"""
    return {'fp': _fp(t), 'full': t.detach().cpu().clone() if t.numel() * t.element_size() <= FULL_LIMIT else None}


def _taps(eng):
    """every tap of the workspace in op order, activation and gradient, as raw bytes"""
    out = {}
    esz = 2 if eng.act_dtype == torch.bfloat16 else 4
    for name, (dims, off, isf, goff) in eng.taps().items():
        nb = int(np.prod(dims)) * (4 if isf else esz)
        out[name] = _fp(eng.ws[off:off + nb])
        if goff >= 0:
            out[name + ' (grad)'] = _fp(eng.ws[goff:goff + nb])
    return out


def _leaves(eng, flat):
    return {name: _fp(flat[off:off + int(np.prod(shape))]) for name, (shape, off) in eng.spec.items()}


SAMPLE = 1024       # elements of each leaf kept (evenly spaced, the same in every child) to bound the differences per leaf


def _samples(eng, flat):
    out = {}
    for name, (shape, off) in eng.spec.items():
        n = int(np.prod(shape))
        idx = torch.linspace(0, n - 1, min(n, SAMPLE), device=flat.device).round().long() + off
        out[name] = flat[idx].cpu()
    return out


def _inputs(B, S, seed):
    from novel_view_synthesis_3d_b200.synthetic import synthetic_batch
    batch, noise = synthetic_batch(B, S, seed=seed)
    mask = np.array([1.0, 0.0, 1.0, 1.0] * B, np.float32)[:B]
    return batch, noise, mask


def _model(plan):
    import novel_view_synthesis_3d_b200 as P
    preset, S, B, dtype, training = L.PLANS[plan]
    cfg = dataclasses.replace(getattr(P, preset), dtype='bf16' if dtype == 1 else 'fp32')
    return P.XUNet.from_config(cfg), S, B, training


def _train_plan(plan, graph, extras):
    import novel_view_synthesis_3d_b200 as P
    model, S, B, _ = _model(plan)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, init_on_device=True)
    step = P.TrainStep(st, use_graph=graph)
    eng = step.eng
    eng.ws.zero_()
    batch, noise, mask = _inputs(B, S, 100 + S + B)
    loss = step(batch, noise, cond_mask=mask)
    torch.cuda.synchronize()
    r = {'loss': _rec(loss.reshape(1)), 'eps': _rec(eng.eps), 'taps': _taps(eng), 'grads': _leaves(eng, eng.grads),
         'params': _leaves(eng, st.params.flat), 'grads_full': _rec(eng.grads), 'params_full': _rec(st.params.flat),
         'grads_s': _samples(eng, eng.grads), 'params_s': _samples(eng, st.params.flat)}
    if extras:
        # the input / camera VJP of a fresh forward, then a k = 2 accumulation pair, on the step's inputs
        flat = st.params.flat
        d_eps = torch.randn(eng.eps.shape, generator=torch.Generator(device=eng.device).manual_seed(5), device=eng.device)
        eng.forward(flat, train=True, seed=7)
        grads, out = eng.backward_vjp_inputs(flat, d_eps, dx=True, dz=True, cameras=True)
        torch.cuda.synchronize()
        r['vjp_grads'] = _rec(grads)
        r.update({f'vjp_{k}': _rec(v) for k, v in out.items()})
        eng.forward(flat, train=True, seed=8)
        eng.backward(flat)
        eng.forward(flat, train=True, seed=9)
        loss2, grads = eng.backward(flat, accumulate=True)
        torch.cuda.synchronize()
        r['accum_grads'] = _rec(grads)
        r['accum_loss'] = _rec(loss2)
    del step, st, eng, model
    return r


def _sampler_plan(plan, graph):
    import novel_view_synthesis_3d_b200 as P
    model, S, B, _ = _model(plan)
    views = B // 2
    params = model.init({'params': 3}, {'x': np.zeros((B, S, S, 3), np.float32)}, zero_init=False, on_device=True)['params']
    smp = P.Sampler(model, params, views, S, steps=256, w=3.0, use_graph=graph)
    smp.eng.ws.zero_()
    batch, _, _ = _inputs(views, S, 200 + views)
    smp.capture(batch)                  # three steps, static conditioning after the first
    torch.cuda.synchronize()
    r = {'z': _rec(smp.z), 'eps': _rec(smp.eng.eps), 'taps': _taps(smp.eng)}
    del smp, params, model
    return r


class _SnapshotReducer:
    """Stands in for dist.GradReducer in a TrainStep: on_bucket enqueues a copy of the bucket on the current stream"""
    enabled = True

    def __init__(self, grads):
        self.flat, self.snap, self.ranges = grads, torch.full_like(grads, float('nan')), []

    def begin(self):
        self.ranges = []

    def on_bucket(self, off, n):
        self.ranges.append((off, n))
        self.snap[off:off + n].copy_(self.flat[off:off + n])

    def wait(self):
        pass


def _bucket_result(snap, grads, ranges):
    n = grads.numel()
    cover = sorted(ranges)
    tiled = bool(cover) and cover[0][0] == 0 and sum(c[1] for c in cover) == n and \
        all(a[0] + a[1] == b[0] for a, b in zip(cover, cover[1:]))
    bad = [(o, m) for o, m in ranges if not torch.equal(snap[o:o + m].view(torch.int32), grads[o:o + m].view(torch.int32))]
    return {'buckets': len(ranges), 'tiled': tiled, 'stale': bad}


def _buckets_engine(plan, min_bytes, graph):
    """forward + backward on the engine with the snapshot hook installed, eager or replayed from a captured graph"""
    import novel_view_synthesis_3d_b200 as P
    model, S, B, _ = _model(plan)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, init_on_device=True)
    eng = model.engine(B, S, True)
    batch, noise, mask = _inputs(B, S, 300 + S)
    eng.load_inputs(batch, cond_mask=mask, noise=noise)
    red = _SnapshotReducer(eng.grads)
    eng.set_bucket_callback(red.on_bucket, min_bytes)
    flat = st.params.flat
    try:
        def fb():
            red.begin()
            eng.forward(flat, train=True, seed=21)
            eng.backward(flat)
        if graph:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fb()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                fb()
            red.snap.fill_(float('nan'))
            eng.grads.fill_(float('nan'))
            g.replay()
        else:
            fb()
        torch.cuda.synchronize()
        r = _bucket_result(red.snap, eng.grads, red.ranges)
    finally:
        eng.set_bucket_callback(None)
    del eng, st, model
    return r


def _buckets_trainstep(plan, bucket_mb, graph):
    """TrainStep with k = 2 micro-batches: only the second backward carries the hook; the second call of the step (a pure
    replay under graphs) is the one checked"""
    import novel_view_synthesis_3d_b200 as P
    model, S, B, _ = _model(plan)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, init_on_device=True)
    step = P.TrainStep(st, use_graph=graph, grad_accum_steps=2, bucket_mb=bucket_mb)
    red = step.reducer = _SnapshotReducer(step.eng.grads)
    for i in range(2):
        batch, noise, mask = _inputs(2 * B, S, 400 + i)
        red.snap.fill_(float('nan'))
        step(batch, noise, cond_mask=mask)
    torch.cuda.synchronize()
    r = _bucket_result(red.snap, step.eng.grads, red.ranges)
    step.reducer = None
    del step, st, model
    return r


def _variants(log_path, cases):
    """the conv_tc / wgrad_tc lines each plan launch logs, per launch id: launched once more on zero buffers between markers"""
    import tests.test_gpu_plan_launches as TL
    for case in cases:
        os.write(2, f'@@case {case[0]}\n'.encode())
        TL._launch_all_convs([case])
    os.write(2, b'@@end\n')
    out, cur = {}, None
    for line in open(log_path).read().split('@@end\n')[0].splitlines():
        if line.startswith('@@case '):
            cur = line[7:]
            out[cur] = []
        elif cur is not None and (line.startswith('conv_tc mode=') or line.startswith('wgrad_tc ')):
            kv = dict(re.findall(r'(\w+)=(-?\w+)', line))
            kv = {k: int(v) if re.fullmatch(r'-?\d+', v) else v for k, v in kv.items()}
            kv['kind'] = 'conv' if line.startswith('conv_tc') else 'wgrad'
            out[cur].append(kv)
    return out


def _changed(base, now):
    """the variant fields of a launch's log lines that differ from the unreserved run"""
    if len(base) != len(now):
        return ['launch count']
    return sorted({k for a, b in zip(base, now) for k in VARIANT if a.get(k) != b.get(k)})


def _recheck(cases, base, now):
    """test_conv_launch (fp64, per element) again for every launch whose variant changed: {id: (changed fields, {check:
    worst err/bound}, failure or None)}"""
    import tests.test_gpu_plan_launches as TL
    from novel_view_synthesis_3d_b200 import _lib
    lib = _lib.load()
    orig = TL._check
    out = {}
    for case in cases:
        ch = _changed(base[case[0]], now[case[0]])
        if not ch:
            continue
        worst = {}

        def check(name, what, got, ref, bound, worst=worst):
            worst[what] = L.excess(got, ref, bound)[0]
            return orig(name, what, got, ref, bound)
        TL._check = check
        err = None
        try:
            TL.test_conv_launch(lib, case)
        except AssertionError as e:
            err = str(e)[:500]
        finally:
            TL._check = orig
        out[case[0]] = (ch, worst, err)
        torch.cuda.empty_cache()
    return out


def _child(env, plans, recheck_plans, graph, buckets, conv_log, base_variants, out_path, log_path):
    fd = os.open(log_path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
    os.dup2(fd, 2)
    assert all(os.environ.get(k) == env.get(k) for k in SWITCHES), 'the switches must be set before the child starts'
    torch.cuda.set_device(0)
    rec = {'env': env, 'seconds': {}}
    t0 = time.perf_counter()
    if conv_log:
        import tests.test_gpu_plan_launches as TL
        cases = [c for c in TL.CONVS if c[0].split(':')[0] in plans]
        rec['variants'] = _variants(log_path, cases)
        rec['seconds']['variants'] = time.perf_counter() - t0
        if base_variants is not None:
            t1 = time.perf_counter()
            rec['recheck'] = _recheck([c for c in cases if c[0].split(':')[0] in recheck_plans], base_variants, rec['variants'])
            rec['seconds']['recheck'] = time.perf_counter() - t1
    for plan in plans:
        for g in ((False, True) if graph else (False,)):
            t1 = time.perf_counter()
            key = plan + ('@graph' if g else '')
            if L.PLANS[plan][4]:
                rec[key] = _train_plan(plan, g, extras=plan == 'full128' and not g)
            else:
                rec[key] = _sampler_plan(plan, g)
            gc.collect()
            torch.cuda.empty_cache()
            rec['seconds'][key] = time.perf_counter() - t1
    if buckets:
        t1 = time.perf_counter()
        rec['buckets'] = {
            'full128 engine eager, 128 MB': _buckets_engine('full128', 128 << 20, False),
            'full128 engine graph, 128 MB': _buckets_engine('full128', 128 << 20, True),
            'small64 engine eager, 64 KB': _buckets_engine('small64', 64 << 10, False),
            'small64 engine graph, 64 KB': _buckets_engine('small64', 64 << 10, True),
            'small64 TrainStep k=2 eager, 64 KB': _buckets_trainstep('small64', 1 / 16, False),
            'small64 TrainStep k=2 graph, 64 KB': _buckets_trainstep('small64', 1 / 16, True),
            'full128 TrainStep k=2 graph, 128 MB': _buckets_trainstep('full128', 128., True),
        }
        gc.collect()
        torch.cuda.empty_cache()
        rec['seconds']['buckets'] = time.perf_counter() - t1
    torch.save(rec, out_path)


# ======================================================================================================================
# parent side: one child per setting, run once per module
# ======================================================================================================================
def _run_child(tmp, name, env, plans, graph=False, buckets=False, conv_log=False, base_variants=None, recheck=()):
    import torch.multiprocessing as mp
    out, log = os.path.join(tmp, f'{name}.pt'), os.path.join(tmp, f'{name}.log')
    env = dict(env, **({'XUNET_CONV_LOG': '1'} if conv_log else {}))
    saved = {k: os.environ.get(k) for k in SWITCHES}
    ctx = mp.get_context('spawn')
    p = ctx.Process(target=_child, args=(env, plans, recheck, graph, buckets, conv_log, base_variants, out, log))
    t0 = time.perf_counter()
    try:
        # the library reads the switches once per process: the child starts with them in its environment
        for k in SWITCHES:
            os.environ.pop(k, None)
        os.environ.update(env)
        p.start()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    p.join(1800)
    if p.is_alive():
        p.kill()
        p.join()
    dt = time.perf_counter() - t0
    tail = open(log).read()[-3000:] if os.path.exists(log) else ''
    if p.exitcode != 0 or not os.path.exists(out):
        return {'error': f'child {name} exited with {p.exitcode}:\n{tail}', 'wall': dt}
    rec = torch.load(out, weights_only=False)
    rec['wall'] = dt
    print(f'child {name} ({" ".join(f"{k}={v}" for k, v in env.items()) or "defaults"}): {dt:.0f} s; ' +
          ', '.join(f'{k} {v:.0f} s' for k, v in rec['seconds'].items()))
    return rec


@pytest.fixture(scope='module')
def runs(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp('schedules'))
    plans = tuple(L.PLANS)
    out = {'ref': _run_child(tmp, 'ref', REF, plans)}
    out['default'] = _run_child(tmp, 'default', MODES['default'], plans, graph=True, buckets=True, conv_log=True)
    for m in ('no_pdl', 'no_side_stream'):
        out[m] = _run_child(tmp, m, MODES[m], plans)
    base = out['default'].get('variants')
    for k, pl in RESERVES.items():
        out[f'reserve{k}'] = (_run_child(tmp, f'reserve{k}', {'XUNET_SM_RESERVE': str(k)}, pl, conv_log=True, base_variants=base,
                                          recheck=RECHECK[k])
                              if base is not None else {'error': 'the unreserved child logged no variants'})
    return out


def _get(runs, name):
    r = runs[name]
    assert 'error' not in r, r['error']
    return r


def _diff(ref, got):
    """what differs, in this order: loss / eps / z, the taps in op order, then the leaves of the gradient and of the parameters
    and the remaining records; empty when every byte matches"""
    out = []
    for k in ref:
        if k in ('taps', 'grads', 'params', 'grads_s', 'params_s') or (k.startswith(('vjp_', 'accum_')) and k not in got):
            continue        # the VJP and accumulation records come from the eager run only
        a, b = ref[k], got.get(k)
        if b is None or a['fp'] != b['fp']:
            out.append(k)
    first = [t for t in ref['taps'] if ref['taps'][t] != got['taps'].get(t)]
    out += [f'tap {t}' for t in first]
    for part in ('grads', 'params'):
        if part in ref:
            out += [f'{part} leaf {n}' for n in ref[part] if ref[part][n] != got[part].get(n)]
    return out


def _report(diff):
    taps = [d for d in diff if d.startswith('tap ')]
    leaves = [d for d in diff if d.startswith('grads leaf ')]
    records = [d for d in diff if not d.startswith(('tap ', 'grads leaf ', 'params leaf '))]
    return (f'first differing tap in op order: {taps[0][4:] if taps else "none"}; {len(taps)} taps differ; {len(leaves)} '
            f'gradient leaves differ: {[d[11:] for d in leaves[:8]]}; records that differ: {records}')


def _max_rel(ref, got):
    """largest |got - ref| / max|ref| over the records held whole (reported beside a mismatch)"""
    worst = {}
    for k, a in ref.items():
        if isinstance(a, dict) and a.get('full') is not None and got.get(k, {}).get('full') is not None and a['fp'] != got[k]['fp']:
            x, y = a['full'].double(), got[k]['full'].double()
            worst[k] = float((x - y).abs().max() / x.abs().max().clamp_min(1e-30))
    return worst


# ======================================================================================================================
# B: schedule invariance
# ======================================================================================================================
CASES_B = [(m, p, g) for m in MODES for p in L.PLANS for g in ((False, True) if m == 'default' else (False,))]


@pytest.mark.parametrize('mode,plan,graph', CASES_B, ids=[f'{m}-{p}' + ('-graph' if g else '') for m, p, g in CASES_B])
def test_schedule_gives_the_same_bits(runs, mode, plan, graph):
    ref = _get(runs, 'ref')[plan]
    got = _get(runs, mode)[plan + ('@graph' if graph else '')]
    diff = _diff(ref, got)
    print(f'{mode} {plan}{" graph" if graph else ""}: {len(ref["taps"])} taps, {len(ref.get("grads", {}))} leaves: ' +
          ('bit-identical' if not diff else _report(diff)))
    assert not diff, f'{mode} {plan}{" graph" if graph else ""} differs from the serialised step: {_report(diff)}; ' \
                     f'largest relative differences {_max_rel(ref, got)}'


# ======================================================================================================================
# C: gradient buckets are final when they are handed out
# ======================================================================================================================
def test_buckets_are_final_when_handed_out(runs):
    b = _get(runs, 'default')['buckets']
    for name, r in b.items():
        print(f'{name}: {r["buckets"]} buckets, tile the buffer: {r["tiled"]}, stale: {len(r["stale"])}')
    for name, r in b.items():
        assert r['tiled'], f'{name}: the buckets do not tile the gradient buffer'
        assert not r['stale'], f'{name}: {len(r["stale"])} of {r["buckets"]} buckets were handed out before they were final: {r["stale"][:4]}'
    assert b['full128 engine eager, 128 MB']['buckets'] >= 8
    assert b['small64 engine eager, 64 KB']['buckets'] >= 8


# ======================================================================================================================
# D: another SM count
# ======================================================================================================================
@pytest.mark.parametrize('reserve', sorted(RESERVES))
def test_sm_reserve_launches_within_fp64_bounds(runs, reserve):
    r = _get(runs, f'reserve{reserve}')
    rc = r['recheck']
    per_check = {}
    for name, (ch, worst, err) in rc.items():
        for what, v in worst.items():
            per_check[what] = max(per_check.get(what, 0.), v)
    print(f'{132 - reserve} SMs: {len(rc)} of {len(r["variants"])} conv launches changed variant and were re-checked; '
          f'worst err/bound per check: ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(per_check.items())))
    fails = {n: e for n, (_, _, e) in rc.items() if e is not None}
    assert not fails, fails


def test_sm_reserves_reach_new_variants(runs):
    """the reserves reach tile widths, persistent-loop lengths and split factors that the unreserved plans do not have"""
    base = _get(runs, 'default')['variants']
    pairs = {k: [(a, b) for n, v in _get(runs, f'reserve{k}')['variants'].items() for a, b in zip(base[n], v)] for k in RESERVES}
    allp = [ab for v in pairs.values() for ab in v]
    reached = {
        'a persistent conv grid newly shorter than its tiles': any(
            b['kind'] == 'conv' and b['ctas'] < b['tiles'] and not a['ctas'] < a['tiles'] for a, b in allp),
        'a conv BN other than the unreserved one': any(b['kind'] == 'conv' and a['BN'] != b['BN'] for a, b in allp),
        'a new wgrad split-K factor that does not divide the pixel tiles': any(
            b['kind'] == 'wgrad' and b['ptiles'] % b['ksplit'] != 0 and a['ksplit'] != b['ksplit'] for a, b in allp),
        'at 2 SMs, a persistent grid looping over 16 or more tiles per CTA': any(
            b['kind'] == 'conv' and b['tiles'] >= 16 * b['ctas'] for a, b in pairs[130]),
    }
    for k, v in pairs.items():
        print(f'{132 - k} SMs: {sum(a != b for a, b in v)} of {len(v)} logged launches change; BN '
              f'{sorted({(a["BN"], b["BN"]) for a, b in v if b["kind"] == "conv" and a["BN"] != b["BN"]})}, ksplit '
              f'{sorted({(a["ksplit"], b["ksplit"], b["ptiles"]) for a, b in v if b["kind"] == "wgrad" and a["ksplit"] != b["ksplit"]})[:12]}, '
              f'most tiles per CTA {max((b["tiles"] / b["ctas"] for a, b in v if b["kind"] == "conv"), default=0):.0f}')
    for k, v in reached.items():
        print(f'  {k}: {"reached" if v else "NOT reached"}')
    assert all(reached.values()), [k for k, v in reached.items() if not v]


CASES_D = [(k, p) for k, pl in sorted(RESERVES.items()) for p in pl]


@pytest.mark.parametrize('reserve,plan', CASES_D, ids=[f'{k}-{p}' for k, p in CASES_D])
def test_sm_reserve_step(runs, reserve, plan):
    """The whole step at another SM count, against the serialised reference.

    How each reduction is split into fp32 partial sums does not follow the reserve to longer sums: the GroupNorm pixels per
    block, the SIMT and thin weight-gradient splits take the whole device's SM count, and wgrad_tc's split-K factor is never
    below the whole device's.  So:
      * fp32 (small64_f32: no tensor-core kernel) computes the same bits: loss, eps, every tap, gradient and parameter;
      * bf16: a changed conv tile width (BN) can change the order of the wgmma K steps (the halo kernel's channel chunk) and a
        finer wgrad_tc split changes its fp32 partial sums, so bits may differ, by the rounding of those launches, which the
        fp64 re-checks above bound, carried through the rest of the network.  Held per leaf: the gradient sample of each leaf
        within 0.5 of its own norm plus 4e-2 of the mean leaf norm (a zero-gradient leaf, e.g. the key bias, is pure rounding),
        eps and the loss (or z) within rel-L2 4e-2, the bf16 noise floor scale of these networks (tests/test_gpu_round2.py);
        and every updated parameter within 2 lr of the reference: Adam's first step moves a parameter by lr g / (|g| + eps),
        at most lr either way, whatever the gradient.
    The first differing tap in op order is reported."""
    ref = _get(runs, 'ref')[plan]
    got = _get(runs, f'reserve{reserve}')[plan]
    diff = _diff(ref, got)
    bf16 = L.PLANS[plan][3] == 1
    rel = lambda k: float(torch.linalg.norm(got[k]['full'].double() - ref[k]['full'].double()) /
                          torch.linalg.norm(ref[k]['full'].double()))
    outs = ('loss', 'eps') if 'loss' in ref else ('z', 'eps')
    rels = {k: rel(k) for k in outs}
    msg = f'{132 - reserve} SMs {plan}: ' + ('bit-identical' if not diff else _report(diff) + f'; rel-L2 {rels}')
    if 'grads_s' in ref:
        g0, g1 = ref['grads_s'], got['grads_s']
        norms = {n: float(torch.linalg.norm(g0[n].double())) for n in g0}
        mean = float(np.sqrt(np.mean([v * v for v in norms.values()])))
        ratio = {n: float(torch.linalg.norm(g1[n].double() - g0[n].double())) / (0.5 * norms[n] + 4e-2 * mean) for n in g0}
        worst = max(ratio, key=ratio.get)
        p0, p1 = ref['params_s'], got['params_s']
        lr = 1e-4
        pr = {n: float(((p1[n].double() - p0[n].double()).abs() / (2 * lr + 2. ** -22 * p0[n].double().abs())).max()) for n in p0}
        pworst = max(pr, key=pr.get)
        msg += f'; worst gradient leaf {worst} at {ratio[worst]:.3g} of its bound; worst parameter {pworst} at {pr[pworst]:.3g}'
        assert pr[pworst] <= 1., msg
        assert ratio[worst] <= 1., msg
    print(msg)
    if not bf16:
        assert not diff, msg
    assert all(math.isfinite(v) and v <= 4e-2 for v in rels.values()), msg
