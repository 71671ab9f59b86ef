"""Time the wgmma attention backward at the bench shape (op level, CUDA events), for A/B experiments."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from novel_view_synthesis_3d_b200 import _lib
lib = _lib.load()
st = torch.cuda.current_stream().cuda_stream
N, L, C, h = 16, 1024, 64, 4
bf = torch.bfloat16
qkv = torch.randn(N, L, 3 * C, device='cuda').to(bf); res = torch.randn(N, L, C, device='cuda').to(bf)
out = torch.empty_like(res); lse = torch.empty(N, h, L, device='cuda'); d = torch.empty(N * L * (h + C), device='cuda')
dout = torch.randn(N, L, C, device='cuda').to(bf); dqkv = torch.empty_like(qkv)
assert lib.xunet_op_attention(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), lse.data_ptr(), N, L, C, h, 1, st) == 0
f = lambda: lib.xunet_op_attention_bwd(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                       d.data_ptr(), dqkv.data_ptr(), N, L, C, h, 1, st)
for _ in range(5): f()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 50
e0.record()
for _ in range(reps): f()
e1.record(); torch.cuda.synchronize()
print(f'{e0.elapsed_time(e1) / reps * 1e3:.1f} us')
