"""Launch single operators at the bench shapes (for `ncu --set full -k regex:<kernel>` captures)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault('XUNET_OP_CACHE_SHADOW', '1')
import torch
from novel_view_synthesis_3d_b200 import _lib
lib = _lib.load()
st = torch.cuda.current_stream().cuda_stream
N, bf = 16, torch.bfloat16
which = sys.argv[1] if len(sys.argv) > 1 else 'all'
reps = 3
if which in ('attn', 'all'):
    L, C, h = 1024, 64, 4
    qkv = torch.randn(N, L, 3 * C, device='cuda').to(bf); res = torch.randn(N, L, C, device='cuda').to(bf)
    out = torch.empty_like(res); lse = torch.empty(N, h, L, device='cuda'); d = torch.empty(N * L * (h + C), device="cuda")
    dout = torch.randn(N, L, C, device='cuda').to(bf); dqkv = torch.empty_like(qkv)
    for _ in range(reps):
        assert lib.xunet_op_attention(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), lse.data_ptr(), N, L, C, h, 1, st) == 0
        assert lib.xunet_op_attention_bwd(1, 1, qkv.data_ptr(), res.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                          d.data_ptr(), dqkv.data_ptr(), N, L, C, h, 1, st) == 0
if which in ('conv', 'all'):
    for (H, Ci, Co) in ((64, 32, 32), (32, 64, 64)):
        x = torch.randn(N, H, H, Ci, device='cuda').to(bf); w = torch.randn(9 * Ci * Co, device='cuda') * 0.05
        b = torch.zeros(Co, device='cuda'); y = torch.empty(N, H, H, Co, device='cuda', dtype=bf)
        dw = torch.zeros(9 * Ci * Co, device='cuda'); db = torch.zeros(Co, device='cuda')
        for _ in range(reps):
            assert lib.xunet_op_conv(1, 1, x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y.data_ptr(), N, H, H, Ci, Co, 3, 1, 1, 1.0, st) == 0
            assert lib.xunet_op_conv_wgrad(1, 1, x.data_ptr(), y.data_ptr(), dw.data_ptr(), db.data_ptr(), N, H, H, Ci, Co, 3, 1, 1, 1.0, st) == 0
if which in ('full1x1', 'fullshapes'):
    # full-3DiM per-pixel GEMMs (FiLM Dense / skip Dense)
    for (H, Ci, Co) in ((32, 1024, 2048), (128, 1024, 512)):
        Nn = 8
        x = torch.randn(Nn, H, H, Ci, device='cuda').to(bf); w = torch.randn(Ci * Co, device='cuda') * 0.02
        b = torch.zeros(Co, device='cuda'); y = torch.empty(Nn, H, H, Co, device='cuda', dtype=bf)
        for _ in range(reps):
            assert lib.xunet_op_conv(1, 1, x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y.data_ptr(), Nn, H, H, Ci, Co, 1, 1, 1, 1.0, st) == 0
if which in ('fullwgrad', 'fullshapes'):
    for (H, Ci, Co) in ((128, 256, 256), (64, 512, 512)):
        Nn = 8
        x = torch.randn(Nn, H, H, Ci, device='cuda').to(bf); y = torch.randn(Nn, H, H, Co, device='cuda').to(bf)
        dw = torch.zeros(9 * Ci * Co, device='cuda'); db = torch.zeros(Co, device='cuda')
        for _ in range(reps):
            assert lib.xunet_op_conv_wgrad(1, 1, x.data_ptr(), y.data_ptr(), dw.data_ptr(), db.data_ptr(), Nn, H, H, Ci, Co, 3, 1, 1, 1.0, st) == 0
if which in ('full3x3', 'fullshapes'):
    for (H, Ci, Co) in ((128, 256, 256),):
        Nn = 8
        x = torch.randn(Nn, H, H, Ci, device='cuda').to(bf); w = torch.randn(9 * Ci * Co, device='cuda') * 0.02
        b = torch.zeros(Co, device='cuda'); y = torch.empty(Nn, H, H, Co, device='cuda', dtype=bf)
        for _ in range(reps):
            assert lib.xunet_op_conv(1, 1, x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y.data_ptr(), Nn, H, H, Ci, Co, 3, 1, 1, 1.0, st) == 0
torch.cuda.synchronize()
print('done')
