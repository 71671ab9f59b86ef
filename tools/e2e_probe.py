"""Where does the host spend its time in an end-to-end step?  (pinned staging ring / event waits / graph launch / loss copy)
   python tools/e2e_probe.py [steps]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches
B, S, K = 8, 64, int(sys.argv[1]) if len(sys.argv) > 1 else 50
model = P.XUNet(dtype='bf16')
state = P.create_train_state(0, 1, 1e-4, B, S, model=model)
step = P.TrainStep(state)
host = make_host_batches(4, B, S, 1234)
mask = np.ones(B, np.float32)
for i in range(5):
    step(host[i % 4][0], host[i % 4][1], cond_mask=mask)
torch.cuda.synchronize()
eng = step.eng
t_load = t_replay = t_wait = 0.0
orig_sync = torch.cuda.Event.synchronize
def timed_sync(self):
    global t_wait
    t0 = time.perf_counter(); orig_sync(self); t_wait += time.perf_counter() - t0
torch.cuda.Event.synchronize = timed_sync
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t_begin = time.perf_counter(); e0.record()
for i in range(K):
    nb, nz = host[i % 4]
    t0 = time.perf_counter()
    eng.load_inputs(nb, cond_mask=mask, noise=nz)
    t1 = time.perf_counter()
    step.graph_fb.replay()
    t2 = time.perf_counter()
    t_load += t1 - t0; t_replay += t2 - t1
e1.record(); torch.cuda.synchronize()
wall = time.perf_counter() - t_begin
print(f'slots={eng.PIN_SLOTS} steps={K}: wall {wall / K * 1e3:.3f} ms/step, device {e0.elapsed_time(e1) / K:.3f} ms/step; host load_inputs '
      f'{t_load / K * 1e3:.3f} ms (of which event waits {t_wait / K * 1e3:.3f}), graph launch {t_replay / K * 1e3:.3f} ms')
