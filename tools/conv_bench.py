"""wgmma conv kernels at full-3DiM shapes: TFLOP/s of forward, dgrad, wgrad (kernel alone, weights pre-converted)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ['XUNET_OP_CACHE_SHADOW'] = '1'
import torch
from novel_view_synthesis_3d_b200 import _lib
from bench import time_kernel
lib = _lib.load(); st = torch.cuda.current_stream().cuda_stream; bf = torch.bfloat16
N = int(sys.argv[1]) if len(sys.argv) > 1 else 4
for (H, Ci, Co, ks) in ((128, 256, 256, 3), (64, 512, 512, 3), (32, 512, 512, 3), (16, 1024, 1024, 3), (64, 1024, 512, 3), (128, 1024, 512, 1), (32, 1024, 2048, 1)):
    x = torch.randn(N, H, H, Ci, device='cuda').to(bf); w = torch.randn(ks * ks * Ci * Co, device='cuda') * 0.02
    b = torch.zeros(Co, device='cuda'); y = torch.empty(N, H, H, Co, device='cuda', dtype=bf); dx = torch.empty_like(x)
    dw = torch.zeros(ks * ks * Ci * Co, device='cuda'); db = torch.zeros(Co, device='cuda')
    fl = 2.0 * N * H * H * ks * ks * Ci * Co
    f = lambda: lib.xunet_op_conv(1, 1, x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y.data_ptr(), N, H, H, Ci, Co, ks, 1, 1, 1.0, st)
    g = lambda: lib.xunet_op_conv_dgrad(1, 1, y.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, H, Ci, Co, ks, 1, 1, 1.0, 0, st)
    h = lambda: lib.xunet_op_conv_wgrad(1, 1, x.data_ptr(), y.data_ptr(), dw.data_ptr(), db.data_ptr(), N, H, H, Ci, Co, ks, 1, 1, 1.0, st)
    assert f() == 0 and g() == 0 and h() == 0, lib.xunet_last_error()
    tf, tg, th = time_kernel(f, 20, 3), time_kernel(g, 20, 3), time_kernel(h, 20, 3)
    print(f'N={N} {H}x{H} {Ci}->{Co} k{ks}: fwd {tf*1e6:8.1f} us {fl/tf/1e12:7.1f} TF/s | dgrad {tg*1e6:8.1f} us {fl/tg/1e12:7.1f} | wgrad {th*1e6:8.1f} us {fl/th/1e12:7.1f}')
