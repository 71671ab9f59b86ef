"""Host cost of replaying the captured forward and backward graphs of the training plan."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches

B, S = 8, 64
host = make_host_batches(1, B, S, 1234)
model = P.XUNet(dtype='bf16')
state = P.create_train_state(0, 1, 1e-4, B, S, model=model)
eng = model.engine(B, S, True)
eng.load_inputs(host[0][0], cond_mask=np.ones(B, np.float32), noise=host[0][1])
flat = state.params.flat
nf, nb = eng.count_kernels(flat)
graphs = {}
st = torch.cuda.Stream()
for name, fn in (('fwd', lambda: eng.forward(flat, train=True)), ('bwd', lambda: eng.backward(flat))):
    with torch.cuda.stream(st):
        eng.forward(flat, train=True); fn(); st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            fn()
    torch.cuda.synchronize()
    graphs[name] = g
for name, g in graphs.items():
    for _ in range(5): g.replay()
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(20): g.replay()
    t1 = time.perf_counter(); torch.cuda.synchronize(); t2 = time.perf_counter()
    print(f'{name}: kernels fwd/bwd {nf}/{nb}  host {1e3*(t1-t0)/20:.3f} ms/replay  total {1e3*(t2-t0)/20:.3f} ms')
