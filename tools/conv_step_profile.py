"""Per-launch time and TFLOP/s of every wgmma conv launch (forward + data gradient) inside ONE eager training step, matched to
its shape and epilogue variant (EPI, from the kernel's template arguments).  The library logs each launch configuration to stderr with XUNET_CONV_LOG=1 (in launch order); CUPTI (torch.profiler)
gives the device time of the conv_tc_kernel launches in the same order.
   XU_MODEL=full XU_B=4 XU_S=128 python tools/conv_step_profile.py > conv_step_profile.txt"""
import os, re, subprocess, sys, collections
if os.environ.get('XU_CHILD') != '1':
    env = dict(os.environ, XU_CHILD='1', XUNET_CONV_LOG='1', XUNET_NO_PDL='1', XUNET_NO_SIDE_STREAM='1')
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True)
    logs = [l for l in r.stderr.splitlines() if l.startswith('conv_tc mode=')]
    times = [float(l.split()[1]) for l in r.stdout.splitlines() if l.startswith('T ')]
    epis = [l.split()[2] for l in r.stdout.splitlines() if l.startswith('T ')]
    marks = [i for i, l in enumerate(r.stderr.splitlines()) if l.startswith('conv_tc mode=') or l.startswith('MARK')]
    # keep only the log lines of the profiled step (after the last MARK)
    lines = r.stderr.splitlines()
    last = max(i for i, l in enumerate(lines) if l.startswith('MARK'))
    logs = [l for l in lines[last:] if l.startswith('conv_tc mode=')]
    if os.environ.get('XU_KERNEL') == 'wgrad':
        # weight-gradient launches instead (same matching, their own log line)
        logs = [l for l in lines[last:] if l.startswith('wgrad_tc ')]
        print(f'{len(logs)} logged wgrad launches, {len(times)} timed wgrad_tc kernels')
        if len(logs) != len(times):
            print(r.stderr[-2000:]); sys.exit(1)
        agg = collections.OrderedDict()
        for l, t in zip(logs, times):
            kv = dict(re.findall(r'(\w+)=(-?\d+)', l))
            H = int(l.split()[2].split('x')[0])
            N, Ci, Co, ks = int(kv['N']), int(kv['Ci']), int(kv['Co']), int(kv['ks'])
            flops = 2.0 * N * H * H * ks * ks * Ci * Co
            key = (H, Ci, Co, ks, kv['mt'], kv['ksplit'], kv['tm'], kv['tn'], kv['stages'])
            a = agg.setdefault(key, [0, 0.0, flops])
            a[0] += 1; a[1] += t
        tot = sum(a[1] for a in agg.values())
        print('HxH Ci->Co k | mt ksplit tiles_m tiles_n stages | launches  avg us  TFLOP/s  share')
        for key, (n, t, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            H, Ci, Co, ks, mt, ksp, tm, tn, st = key
            print(f'{H:3d}x{H:<3d} {Ci:4d}->{Co:<4d} k{ks} | mt {mt} ksplit {ksp:>2} tm {tm:>3} tn {tn} st {st} | {n:3d}  {t / n:8.1f}  {fl / (t / n) / 1e6:7.1f}  {t / tot * 100:5.1f}%')
        print(f'total wgrad_tc time {tot / 1e3:.2f} ms')
        sys.exit(0)
    print(f'{len(logs)} logged conv launches, {len(times)} timed conv_tc kernels')
    if len(logs) != len(times):
        print(r.stderr[-2000:])
        sys.exit(1)
    agg = collections.OrderedDict()
    for l, t, epi in zip(logs, times, epis):
        kv = dict(re.findall(r'(\w+)=(-?\d+)', l))
        N, H, W = int(kv['N']), int(l.split()[3].split('x')[0]), int(l.split()[3].split('x')[1])
        Ci, Co, ks = int(kv['Ci']), int(kv['Co']), int(kv['ks'])
        flops = 2.0 * N * H * W * ks * ks * Ci * Co
        key = (kv['mode'], epi, H, Ci, Co, ks, kv['BN'], kv['tiles'], kv['ctas'], kv['halo'])
        a = agg.setdefault(key, [0, 0.0, flops])
        a[0] += 1; a[1] += t
    tot = sum(a[1] for a in agg.values())
    print('mode(0 fwd,1 dgrad) EPI HxH Ci->Co k | BN tiles ctas halo | launches  avg us  TFLOP/s  share')
    for key, (n, t, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        mode, epi, H, Ci, Co, ks, BN, tiles, ctas, halo = key
        print(f'{mode} {epi} {H:3d}x{H:<3d} {Ci:4d}->{Co:<4d} k{ks} | BN {BN:>3} tiles {tiles:>5} ctas {ctas:>3} halo {halo} | {n:3d}  {t / n:8.1f}  {fl / (t / n) / 1e6:7.1f}  {t / tot * 100:5.1f}%')
    print(f'total conv_tc time {tot / 1e3:.2f} ms')
    for e in sorted(set(epis)):
        n, t = sum(1 for x in epis if x == e), sum(t for t, x in zip(times, epis) if x == e)
        print(f'EPI {e}: {n} launches, {t / 1e3:.3f} ms')
    sys.exit(0)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches
from torch.profiler import profile, ProfilerActivity
B, S = int(os.environ.get('XU_B', 8)), int(os.environ.get('XU_S', 64))
full = os.environ.get('XU_MODEL', 'small') == 'full'
model = P.XUNet.from_config(P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'})) if full else P.XUNet(dtype='bf16')
state = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=full)
step = P.TrainStep(state, use_graph=False)
host = make_host_batches(1, B, S, 1234)
mask = np.ones(B, np.float32)
for i in range(3):
    step(host[0][0], host[0][1], cond_mask=mask)
torch.cuda.synchronize()
print('MARK', file=sys.stderr, flush=True)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step(host[0][0], host[0][1], cond_mask=mask)
    torch.cuda.synchronize()
kname = 'wgrad_tc_kernel' if os.environ.get('XU_KERNEL') == 'wgrad' else 'conv_tc_kernel'
evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and kname in e.name]
evs.sort(key=lambda e: e.time_range.start)
for e in evs:
    # conv_tc_kernel<BK, EPI, BN>: the second template argument is the epilogue variant (wgrad: '-')
    m = re.search(r'conv_tc_kernel<\d+, (\d+), \d+>', e.name)
    print('T', e.device_time, m.group(1) if m else '-')
