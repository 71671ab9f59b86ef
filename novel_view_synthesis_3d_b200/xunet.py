"""Host-side mirror of the reference's Flax API for the X-UNet (model/xunet.py:205-280).

    model = XUNet()                                            # model/xunet.py:205-215 attributes
    params = model.init({'params': key, 'dropout': key}, sample, cond_mask=np.zeros(B), train=True)['params']
    eps = model.apply({'params': params}, batch, cond_mask=mask, train=True, rngs={'dropout': key})

All compute runs in libxunet_b200.so (hand-written sm_90a CUDA); PyTorch is used only for device memory,
streams and torch.distributed.  There is no CPU / eager fallback: without the library or a GPU this raises.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib

POSE_EMB_DIM = 144
BATCH_KEYS = ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K')
CAMERA_KEYS = ('R1', 't1', 'R2', 't2', 'K')
INPUT_ORDER = BATCH_KEYS + ('cond_mask', 'noise', 'loss_weight')     # segment order of Engine.inp_all
LOSSES = ('frobenius', 'mse')


def check_loss(loss) -> str:
    """Validates a training-loss name: 'frobenius' (the reference's ||eps_hat - noise||_F) or 'mse' (mean squared error)."""
    if loss not in LOSSES:
        raise ValueError(f'loss must be one of {LOSSES}, got {loss!r}')
    return loss


@dataclass(frozen=True)
class XUNetConfig:
    """The nine XUNet attributes of model/xunet.py:207-215 (+ the two implementation knobs)."""
    ch: int = 32
    ch_mult: Tuple[int, ...] = (1, 2)
    emb_ch: int = 32
    num_res_blocks: int = 2
    attn_resolutions: Tuple[int, ...] = (8, 16, 32)
    attn_heads: int = 4
    dropout: float = 0.1
    use_pos_emb: bool = False
    use_ref_pose_emb: bool = False
    dtype: str = 'bf16'                 # 'bf16' (activations bf16, fp32 accumulate) | 'fp32' (exact-fp32 verify mode)
    ray_convention: str = 'v3d130_ij'   # see SURVEY 8(c): visu3d 1.3.0 pixel convention

    def c_struct(self) -> _lib.XunetConfig:
        c = _lib.XunetConfig()
        c.ch = self.ch
        c.n_levels = len(self.ch_mult)
        for i, m in enumerate(self.ch_mult):
            c.ch_mult[i] = m
        c.emb_ch = self.emb_ch
        c.num_res_blocks = self.num_res_blocks
        c.n_attn_resolutions = len(self.attn_resolutions)
        for i, r in enumerate(self.attn_resolutions):
            c.attn_resolutions[i] = r
        c.attn_heads = self.attn_heads
        c.dropout = float(self.dropout)
        c.use_pos_emb = int(self.use_pos_emb)
        c.use_ref_pose_emb = int(self.use_ref_pose_emb)
        c.ray_convention = _lib.RAYS[self.ray_convention]
        return c


# named presets for BASELINE.json's configs
SMALL = XUNetConfig()
FULL_3DIM = XUNetConfig(ch=256, ch_mult=(1, 2, 2, 4), emb_ch=1024, num_res_blocks=3, attn_resolutions=(8, 16, 32),
                        attn_heads=8)


class ParamTree(dict):
    """Nested dict of parameter leaves in the Flax tree shape (SURVEY Appendix A).  `.flat` is the single fp32
    device buffer all leaves are views of (one gradient bucket / one Adam launch)."""
    flat: torch.Tensor = None
    spec: "OrderedDict[str, Tuple[Tuple[int, ...], int]]" = None


def _nest(flat: Dict[str, torch.Tensor]) -> dict:
    tree: dict = {}
    for k, v in flat.items():
        node = tree
        parts = k.split('/')
        for part in parts[:-1]:
            node = node.setdefault(part, {})
        node[parts[-1]] = v
    return tree


def _flatten(tree: dict, prefix='') -> Dict[str, object]:
    out = {}
    for k, v in tree.items():
        if isinstance(v, dict):
            out.update(_flatten(v, prefix + k + '/'))
        else:
            out[prefix + k] = v
    return out


def pack_flat(params: dict, spec, nparams: int) -> torch.Tensor:
    """Nested dict of arrays in the Flax tree shape -> host fp32 flat buffer laid out by `spec` ({name: (shape, offset)}).
    Raises KeyError on missing / unexpected leaves and ValueError on a shape mismatch.  Needs no GPU."""
    leaves = _flatten(params)
    missing = set(spec) - set(leaves)
    extra = set(leaves) - set(spec)
    if missing or extra:
        raise KeyError(f'parameter tree mismatch: missing {sorted(missing)[:3]}..., unexpected {sorted(extra)[:3]}...')
    host = torch.empty(nparams, dtype=torch.float32)
    for name, (shape, off) in spec.items():
        v = torch.as_tensor(np.asarray(leaves[name]) if not isinstance(leaves[name], torch.Tensor) else leaves[name])
        if tuple(v.shape) != tuple(shape):
            raise ValueError(f'{name}: shape {tuple(v.shape)} != {tuple(shape)}')
        host[off: off + v.numel()] = v.reshape(-1).to(torch.float32).cpu()
    return host


def is_zero_init_kernel(name: str) -> bool:
    """out_init_scale() leaves (model/xunet.py:11-12): every ResnetBlock's Conv_1 (:85-89) and the top-level Conv_1
    (:276-280).  NOT 'ConditioningProcessor_0/Conv_1/kernel' -- the level-1 pose-embedding conv (:197-202) keeps the
    default lecun_normal although its auto-name also ends in Conv_1."""
    return name.endswith('Conv_1/kernel') and not name.startswith('ConditioningProcessor_0/')


def _seed_of(key, default=0) -> int:
    if key is None:
        return default
    if isinstance(key, (int, np.integer)):
        return int(key)
    arr = np.asarray(key).reshape(-1)           # e.g. a jax PRNGKey-like uint32[2]
    hi = int(arr[-2]) if arr.size > 1 else 0
    return ((hi << 32) | (int(arr[-1]) & 0xFFFFFFFF)) & 0x7FFFFFFFFFFFFFFF


class InputSlots:
    """Static device inputs of k batches of B samples (k micro-batches of one gradient-accumulation step; k = 1: the engine's
    own inputs).  Slot j holds rows [j*B, (j+1)*B) of a k*B batch and has its own xunet_batch of device pointers.  All slots
    live in ONE device buffer (and one pinned mirror), 256-byte aligned segments in INPUT_ORDER, slot after slot: a training
    step stages every slot with a single H2D copy instead of ten small ones per slot (each costs ~7 us of stream time)."""
    PIN_SLOTS = 3

    def __init__(self, B: int, S: int, k: int, device):
        self.B, self.k = B, k
        f32 = dict(dtype=torch.float32, device=device)
        self.shapes = {'x': (B, S, S, 3), 'z': (B, S, S, 3), 'logsnr': (B,), 'R1': (B, 3, 3), 't1': (B, 3), 'R2': (B, 3, 3),
                       't2': (B, 3), 'K': (B, 3, 3), 'cond_mask': (B,), 'noise': (B, S, S, 3), 'loss_weight': (B,)}
        self._seg, off = {}, 0          # (slot, key) -> (offset, elements)
        for j in range(k):
            for key in INPUT_ORDER:
                n = int(np.prod(self.shapes[key]))
                self._seg[j, key] = (off, n)
                off += (n + 63) // 64 * 64
        self.all = torch.zeros(off, **f32)
        self.inp = [{key: self.all[o:o + n].view(self.shapes[key]) for key in INPUT_ORDER for o, n in [self._seg[j, key]]}
                    for j in range(k)]
        for d in self.inp:
            d['cond_mask'].fill_(1.0)
            d['loss_weight'].fill_(1.0)
        # pinned staging ring: the host may run several steps ahead of the GPU (a step is a few ms of device time, the host
        # side far less), so a slot is rewritten only after the H2D copy that last read it has completed (one event per slot)
        self._pin_ring = [torch.zeros(off, dtype=torch.float32).pin_memory() for _ in range(self.PIN_SLOTS)]
        self._pin_np = [t.numpy() for t in self._pin_ring]      # numpy views of the same pinned memory
        self._pin_events = [None] * self.PIN_SLOTS
        self._pin_next = 0
        self.cbatch = [_lib.XunetBatch(**{key: d[key].data_ptr() for key in BATCH_KEYS + ('cond_mask',)}, rays=None)
                       for d in self.inp]

    def load(self, batch: dict, cond_mask=None, noise=None, loss_weight=None) -> int:
        """Copies one batch dict of k*B samples (numpy / torch, any float dtype) into the slots, micro-batch j into slot j;
        cond_mask, noise and the per-sample loss weights too when given.  Returns the number of host->device bytes moved."""
        k = self.k
        nbytes = 0
        items = [(key, batch[key]) for key in BATCH_KEYS]
        if cond_mask is not None:
            items.append(('cond_mask', cond_mask))
        if noise is not None:
            items.append(('noise', noise))
        if loss_weight is not None:
            items.append(('loss_weight', loss_weight))
        staged = []
        slot, pin = None, None
        for key, v in items:
            shape = self.shapes[key]
            if isinstance(v, torch.Tensor) and v.is_cuda:
                v = v.reshape((k,) + shape)
                for j in range(k):
                    self.inp[j][key].copy_(v[j].to(torch.float32), non_blocking=True)
                continue
            src = (v.detach().float() if v.dtype == torch.bfloat16 else v.detach()).numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
            full = (k * shape[0],) + shape[1:]
            if tuple(src.shape) != full and src.size != k * int(np.prod(shape)):
                raise ValueError(f"batch['{key}'] has shape {tuple(src.shape)}, expected {full}")
            if pin is None:
                slot = self._pin_next
                self._pin_next = (slot + 1) % self.PIN_SLOTS
                if self._pin_events[slot] is not None:
                    self._pin_events[slot].synchronize()      # the copy that last read this slot has finished
                pin = self._pin_ring[slot]
            # float64 -> float32 down-cast (as JAX does with x64 off) straight into pinned memory.  numpy, not torch: a torch CPU
            # copy_ of ~1e5 elements fans out over every host core (3.5 ms on 8 threads against 0.1 ms single-threaded)
            rows = src.reshape(k, -1)
            for j in range(k):
                o, n = self._seg[j, key]
                np.copyto(self._pin_np[slot][o:o + n], rows[j], casting='unsafe')
                staged.append(j * len(INPUT_ORDER) + INPUT_ORDER.index(key))
                nbytes += n * 4
        # one async H2D copy per run of adjacent segments (a full training batch = one copy)
        idx = sorted(staged)
        seg = lambda i: self._seg[i // len(INPUT_ORDER), INPUT_ORDER[i % len(INPUT_ORDER)]]
        i = 0
        while i < len(idx):
            j = i
            while j + 1 < len(idx) and idx[j + 1] == idx[j] + 1:
                j += 1
            lo = seg(idx[i])[0]
            o, n = seg(idx[j])
            self.all[lo:o + n].copy_(pin[lo:o + n], non_blocking=True)
            i = j + 1
        if pin is not None:
            ev = self._pin_events[slot] or torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.all.device))
            self._pin_events[slot] = ev
        return nbytes


class Engine:
    """One compiled execution plan: (config, B, S, training).  Owns the workspace and static I/O buffers."""
    PIN_SLOTS = InputSlots.PIN_SLOTS

    def __init__(self, cfg: XUNetConfig, B: int, S: int, training: bool, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('novel_view_synthesis_3d_b200 needs a CUDA device (H100, sm_90a); there is no CPU path')
        self.lib = _lib.load()
        self.cfg, self.B, self.S, self.training = cfg, B, S, training
        self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
        self.dtype_code = {'fp32': _lib.DTYPE_F32, 'bf16': _lib.DTYPE_BF16}[cfg.dtype]
        self.act_dtype = torch.float32 if cfg.dtype == 'fp32' else torch.bfloat16
        h = C.c_void_p()
        cs = cfg.c_struct()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.xunet_create(C.byref(cs), B, S, self.dtype_code, int(training), C.byref(h)), 'xunet_create')
        self.h = h
        self.nparams = int(self.lib.xunet_param_count(h))
        self.spec = OrderedDict()
        name, ndim, shape, off = C.c_char_p(), C.c_int(), (C.c_longlong * 5)(), C.c_longlong()
        for i in range(self.lib.xunet_param_leaves(h)):
            _lib.check(self.lib.xunet_param_leaf(h, i, C.byref(name), C.byref(ndim), C.byref(shape), C.byref(off)), 'param_leaf')
            self.spec[name.value.decode()] = (tuple(int(shape[k]) for k in range(ndim.value)), int(off.value))
        self.ws_bytes = int(self.lib.xunet_workspace_bytes(h))
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=self.device)
        f32 = dict(dtype=torch.float32, device=self.device)
        self.inputs = InputSlots(B, S, 1, self.device)
        self.inp_all, self.inp, self.cbatch = self.inputs.all, self.inputs.inp[0], self.inputs.cbatch[0]
        self.rays = None          # optional (B,2,S,S,6) device tensor: explicit-rays entry (set_rays)
        self.eps = torch.zeros(B, S, S, 3, **f32)
        self.loss = torch.zeros(1, **f32)
        self.seed = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.grads = torch.zeros(self.nparams, **f32) if training else None
        self.dx = self.dz = None  # backward_vjp's input gradients (B,S,S,3), allocated at the first call that asks for them
        self.cam_grads = {}       # backward_vjp_inputs' ray / camera gradients by name, allocated at the first call that asks
        self._fwd_rays = None     # the explicit rays of the last forward (kept alive for the ray gradient of its VJP)
        self.forward_count = 0    # forwards run so far: a VJP taken later checks that its forward is still the last one
        self._taps = None
        self._bucket_cb = None    # keeps the ctypes callback object alive while it is installed

    def __del__(self):
        try:
            if getattr(self, 'h', None):
                self.lib.xunet_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ---- host -> device staging (pinned memory, async on the current stream) -------------------------
    def load_inputs(self, batch: dict, cond_mask=None, noise=None, loss_weight=None) -> int:
        """Copies one batch dict (numpy / torch, any float dtype) into the static device buffers.
        Returns the number of host->device bytes moved."""
        return self.inputs.load(batch, cond_mask=cond_mask, noise=noise, loss_weight=loss_weight)

    def set_rays(self, rays) -> None:
        """Explicit-rays entry (SURVEY 8(c)): `rays` = (B, 2, S, S, 6) [pos xyz | dir xyz] for camera 1 / camera 2, e.g. the
        output of the reference's own v3d.Camera(...).rays() (model/xunet.py:159-161,166-168); None restores the
        library's ray generation from R, t, K and cfg.ray_convention."""
        if rays is None:
            self.rays = None
            self.cbatch.rays = None
            return
        r = torch.as_tensor(np.asarray(rays) if not isinstance(rays, torch.Tensor) else rays).to(torch.float32)
        if tuple(r.shape) != (self.B, 2, self.S, self.S, 6):
            raise ValueError(f'rays has shape {tuple(r.shape)}, expected {(self.B, 2, self.S, self.S, 6)}')
        self.rays = r.to(self.device).contiguous()
        self.cbatch.rays = self.rays.data_ptr()

    def set_bucket_callback(self, fn, min_bucket_bytes: int = 0) -> int:
        """Installs fn(elem_offset, n_elems), called on the host during backward() whenever a contiguous range of the flat
        gradient buffer is final (see xunet_set_grad_bucket_callback).  fn=None removes it.  Returns the bucket count."""
        if fn is None:
            _lib.check(self.lib.xunet_set_grad_bucket_callback(self.h, _lib.BUCKET_FN(0), None, 0), 'bucket_callback')
            self._bucket_cb = None
            return 0
        cb = _lib.BUCKET_FN(lambda user, off, n: fn(int(off), int(n)))
        _lib.check(self.lib.xunet_set_grad_bucket_callback(self.h, cb, None, int(min_bucket_bytes)), 'bucket_callback')
        self._bucket_cb = cb
        return int(self.lib.xunet_grad_bucket_count(self.h))

    def forward(self, flat_params: torch.Tensor, *, train: bool, seed: Optional[int] = None,
                inputs: Optional[Tuple[InputSlots, int]] = None, seed_dev: Optional[torch.Tensor] = None,
                batch: Optional[_lib.XunetBatch] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """inputs=(slots, j): read slot j of `slots` instead of the engine's own inputs; batch: an xunet_batch of device
        pointers to read instead of either; seed_dev: a device int64 to read the dropout seed from instead of `self.seed`
        (all default to the engine's own buffers).  out: a contiguous fp32 device tensor of `self.eps`'s shape to write the
        output to instead of `self.eps`.  Returns the output."""
        assert flat_params.dtype == torch.float32 and flat_params.is_cuda and flat_params.numel() == self.nparams
        if out is not None and not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()
                                    and out.shape == self.eps.shape):
            raise ValueError(f'out must be a contiguous fp32 device tensor of shape {tuple(self.eps.shape)}')
        if seed is not None:
            self.seed.fill_(int(seed) & 0x7FFFFFFFFFFFFFFF)
        cb = batch if batch is not None else self.cbatch if inputs is None else inputs[0].cbatch[inputs[1]]
        sd = self.seed if seed_dev is None else seed_dev
        st = torch.cuda.current_stream(self.device).cuda_stream
        y = self.eps if out is None else out
        self.forward_count += 1
        self._fwd_rays = self.rays if inputs is None and batch is None else None
        _lib.check(self.lib.xunet_forward(self.h, flat_params.data_ptr(), C.byref(cb), int(train),
                                          sd.data_ptr(), self.ws.data_ptr(), y.data_ptr(), st), 'xunet_forward')
        return y

    def backward(self, flat_params: torch.Tensor, *, accumulate: bool = False, inputs: Optional[Tuple[InputSlots, int]] = None,
                 seed_dev: Optional[torch.Tensor] = None, loss_out: Optional[torch.Tensor] = None, loss: str = 'frobenius',
                 loss_weight: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """The loss and its parameter gradient (train.py:62-71); follows forward() with the same `inputs` and `seed_dev`.
        loss='frobenius': ||eps - noise||_F (train.py:67); loss='mse': (1/B) sum_b w_b * mean_i (eps - noise)_bi^2
        (xunet_backward_mse), with w = loss_weight, a device fp32 (B,) tensor, or all 1 when None.
        accumulate=True adds the gradient into `self.grads` instead of overwriting it.
        loss_out: a device float to write the loss to instead of `self.loss`."""
        if not self.training:
            raise RuntimeError('engine was built with training=False')
        check_loss(loss)
        cb, noise = (self.cbatch, self.inp['noise']) if inputs is None else (inputs[0].cbatch[inputs[1]], inputs[0].inp[inputs[1]]['noise'])
        sd = self.seed if seed_dev is None else seed_dev
        out = self.loss if loss_out is None else loss_out
        st = torch.cuda.current_stream(self.device).cuda_stream
        args = (flat_params.data_ptr(), C.byref(cb), noise.data_ptr())
        tail = (sd.data_ptr(), self.ws.data_ptr(), self.grads.data_ptr(), out.data_ptr())
        if loss == 'mse':
            w = None
            if loss_weight is not None:
                if not (loss_weight.is_cuda and loss_weight.dtype == torch.float32 and loss_weight.is_contiguous()
                        and tuple(loss_weight.shape) == (self.B,)):
                    raise ValueError(f'loss_weight must be a contiguous fp32 device tensor of shape ({self.B},)')
                w = loss_weight.data_ptr()
            _lib.check(self.lib.xunet_backward_mse(self.h, *args, w, *tail, int(accumulate), st), 'xunet_backward_mse')
            return out, self.grads
        if loss_weight is not None:
            raise ValueError("loss_weight needs loss='mse': the Frobenius loss has no per-sample term to weight")
        fn = self.lib.xunet_backward_accumulate if accumulate else self.lib.xunet_backward
        _lib.check(fn(self.h, *args, *tail, st), 'xunet_backward_accumulate' if accumulate else 'xunet_backward')
        return out, self.grads

    def backward_vjp(self, flat_params: torch.Tensor, d_eps: torch.Tensor, *, accumulate: bool = False, dx: bool = False,
                     dz: bool = False, inputs: Optional[Tuple[InputSlots, int]] = None,
                     seed_dev: Optional[torch.Tensor] = None):
        """Vector-Jacobian product of the last forward (xunet_backward_vjp): d_eps = dL/d(eps_hat), a contiguous fp32 device
        tensor (B,S,S,3).  Returns (self.grads, dx, dz): the parameter gradient (accumulate=True adds into self.grads) and, when
        asked for, dL/dx and dL/dz of the input views in the engine's own (B,S,S,3) buffers, which the next call overwrites
        (None when not asked for).  Follows forward() with the same `inputs` and `seed_dev`, like backward()."""
        shape = self._check_d_eps(d_eps)
        if dx and self.dx is None:
            self.dx = torch.zeros(shape, dtype=torch.float32, device=self.device)
        if dz and self.dz is None:
            self.dz = torch.zeros(shape, dtype=torch.float32, device=self.device)
        cb = self.cbatch if inputs is None else inputs[0].cbatch[inputs[1]]
        sd = self.seed if seed_dev is None else seed_dev
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.xunet_backward_vjp(self.h, flat_params.data_ptr(), C.byref(cb), d_eps.data_ptr(), sd.data_ptr(),
                                               self.ws.data_ptr(), self.grads.data_ptr(), int(accumulate),
                                               self.dx.data_ptr() if dx else None, self.dz.data_ptr() if dz else None, st),
                   'xunet_backward_vjp')
        return self.grads, (self.dx if dx else None), (self.dz if dz else None)

    def _check_d_eps(self, d_eps) -> Tuple[int, ...]:
        if not self.training:
            raise RuntimeError('engine was built with training=False')
        shape = (self.B, self.S, self.S, 3)
        if not (isinstance(d_eps, torch.Tensor) and d_eps.is_cuda and d_eps.dtype == torch.float32 and d_eps.is_contiguous()
                and tuple(d_eps.shape) == shape):
            raise ValueError(f'd_eps must be a contiguous fp32 CUDA tensor of shape {shape}')
        return shape

    def backward_vjp_inputs(self, flat_params: torch.Tensor, d_eps: torch.Tensor, *, accumulate: bool = False, dx: bool = False,
                            dz: bool = False, rays: bool = False, cameras: bool = False,
                            inputs: Optional[Tuple[InputSlots, int]] = None, seed_dev: Optional[torch.Tensor] = None):
        """backward_vjp that also differentiates the cameras (xunet_backward_vjp_inputs).  Returns (self.grads, dict): 'x' / 'z'
        when dx / dz, 'rays' = dL/d(rays) (B,2,S,S,6) [pos | dir] of camera 1 / camera 2 when rays or cameras, and 'R1', 't1',
        'R2', 't2', 'K' when cameras (the forward's rays must then have been generated from R, t, K, not given).  The tensors
        are the engine's own buffers, overwritten by the next call.  The parameter gradient, dx and dz are those backward_vjp
        gives, bit for bit.  The log-SNR gets no gradient."""
        shape = self._check_d_eps(d_eps)
        if cameras and self._fwd_rays is not None:
            raise ValueError('camera gradients need rays generated from R, t, K: the forward was given explicit rays')
        sizes = {'x': shape, 'z': shape, 'rays': (self.B, 2, self.S, self.S, 6), 'R1': (self.B, 3, 3), 't1': (self.B, 3),
                 'R2': (self.B, 3, 3), 't2': (self.B, 3), 'K': (self.B, 3, 3)}
        want = [k for k, on in (('x', dx), ('z', dz), ('rays', rays or cameras)) if on] + (list(CAMERA_KEYS) if cameras else [])
        out = {}
        for k in want:
            if k in ('x', 'z'):
                if getattr(self, 'd' + k) is None:
                    setattr(self, 'd' + k, torch.zeros(shape, dtype=torch.float32, device=self.device))
                out[k] = getattr(self, 'd' + k)
            else:
                if k not in self.cam_grads:
                    self.cam_grads[k] = torch.zeros(sizes[k], dtype=torch.float32, device=self.device)
                out[k] = self.cam_grads[k]
        ig = _lib.XunetInputGrads(**{('d_rays' if k == 'rays' else 'd' + k): v.data_ptr() for k, v in out.items()})
        cb = _lib.XunetBatch.from_buffer_copy(self.cbatch if inputs is None else inputs[0].cbatch[inputs[1]])
        cb.rays = self._fwd_rays.data_ptr() if (inputs is None and self._fwd_rays is not None) else None
        sd = self.seed if seed_dev is None else seed_dev
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.xunet_backward_vjp_inputs(self.h, flat_params.data_ptr(), C.byref(cb), d_eps.data_ptr(), sd.data_ptr(),
                                                      self.ws.data_ptr(), self.grads.data_ptr(), int(accumulate), C.byref(ig), st),
                   'xunet_backward_vjp_inputs')
        return self.grads, out

    def count_kernels(self, flat_params: torch.Tensor) -> Tuple[int, int]:
        """(forward, backward) kernel launches of this plan, counted from a throw-away graph capture."""
        nf, nb = C.c_int(0), C.c_int(0)
        g = self.grads.data_ptr() if self.training else None
        _lib.check(self.lib.xunet_count_kernels(self.h, flat_params.data_ptr(), C.byref(self.cbatch), self.inp['noise'].data_ptr(),
                                                self.seed.data_ptr(), self.ws.data_ptr(), g, self.loss.data_ptr(),
                                                C.byref(nf), C.byref(nb)), 'xunet_count_kernels')
        return nf.value, nb.value

    # ---- introspection for parity tests ---------------------------------------------------------------
    def taps(self) -> Dict[str, Tuple[Tuple[int, ...], int, bool, int]]:
        if self._taps is None:
            out = OrderedDict()
            name, dims, off, isf, goff = C.c_char_p(), (C.c_int * 4)(), C.c_longlong(), C.c_int(), C.c_longlong()
            for i in range(self.lib.xunet_tap_count(self.h)):
                _lib.check(self.lib.xunet_tap(self.h, i, C.byref(name), C.byref(dims), C.byref(off), C.byref(isf), C.byref(goff)), 'tap')
                out[name.value.decode()] = (tuple(dims), int(off.value), bool(isf.value), int(goff.value))
            self._taps = out
        return self._taps

    def read_tap(self, name: str, grad: bool = False) -> torch.Tensor:
        dims, off, isf, goff = self.taps()[name]
        if grad:
            if goff < 0:
                raise KeyError(f'{name} has no gradient')
            off = goff
        dt = torch.float32 if isf else self.act_dtype
        n = int(np.prod(dims))
        raw = self.ws[off: off + n * (4 if dt == torch.float32 else 2)]
        return raw.view(dt).reshape(dims).to(torch.float32).clone()


class XUNet:
    """Drop-in for the reference's `XUNet` Flax module as used by train.py:39-43,63-66 and sampling.py:64,100-102,131-132."""

    def __init__(self, ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4,
                 dropout=0.1, use_pos_emb=False, use_ref_pose_emb=False, *, dtype='bf16', ray_convention='v3d130_ij',
                 device=None):
        self.config = XUNetConfig(ch=ch, ch_mult=tuple(ch_mult), emb_ch=emb_ch, num_res_blocks=num_res_blocks,
                                  attn_resolutions=tuple(attn_resolutions), attn_heads=attn_heads, dropout=dropout,
                                  use_pos_emb=use_pos_emb, use_ref_pose_emb=use_ref_pose_emb, dtype=dtype,
                                  ray_convention=ray_convention)
        self.device = device
        self._engines: Dict[Tuple[int, int, bool], Engine] = {}

    @classmethod
    def from_config(cls, cfg: XUNetConfig, device=None) -> "XUNet":
        m = cls.__new__(cls)
        m.config, m.device, m._engines = cfg, device, {}
        return m

    def engine(self, B: int, S: int, training: bool = False) -> Engine:
        key = (B, S, bool(training))
        if key not in self._engines:
            self._engines[key] = Engine(self.config, B, S, training, self.device)
        return self._engines[key]

    # ---- parameters -------------------------------------------------------------------------------------
    def param_spec(self, S: int, B: int = 1) -> "OrderedDict[str, Tuple[Tuple[int, ...], int]]":
        return self.engine(B, S, False).spec

    def tree_from_flat(self, flat: torch.Tensor, S: int, B: int = 1, spec=None) -> ParamTree:
        spec = self.param_spec(S, B) if spec is None else spec
        leaves = {name: flat[off: off + int(np.prod(shape))].view(shape) for name, (shape, off) in spec.items()}
        tree = ParamTree(_nest(leaves))
        tree.flat, tree.spec = flat, spec
        return tree

    def flat_from_tree(self, params, S: int, B: int = 1) -> torch.Tensor:
        """Packs any nested dict of arrays in the Flax tree shape (e.g. an imported checkpoint) into the flat buffer."""
        if isinstance(params, ParamTree) and params.flat is not None:
            return params.flat
        eng = self.engine(B, S, False)
        return pack_flat(params, eng.spec, eng.nparams).to(eng.device)

    def init(self, rngs, batch, *, cond_mask=None, train=True, zero_init=True, on_device=False) -> Dict[str, ParamTree]:
        """Flax-style initialisation (train.py:41-43): lecun_normal kernels, zero biases, GroupNorm scale 1,
        zero-initialised Conv_1 kernels (out_init_scale, model/xunet.py:11-12).  The parameter set depends on the
        image side of `batch['x']` (which levels get attention).  on_device=True draws the same distributions with the
        CUDA generator straight into the flat device buffer (seconds instead of tens of seconds for the 439 M-parameter
        model; a different random stream than the host path)."""
        x = batch['x']
        B, S = int(x.shape[0]), int(x.shape[1])
        eng = self.engine(B, S, False)
        seed = _seed_of(rngs.get('params') if isinstance(rngs, dict) else rngs)
        gdev = eng.device if on_device else 'cpu'
        g = torch.Generator(device=gdev).manual_seed(seed)
        host = torch.zeros(eng.nparams, dtype=torch.float32, device=gdev)
        for name, (shape, off) in eng.spec.items():
            leaf = name.rsplit('/', 1)[-1]
            n = int(np.prod(shape))
            if leaf == 'kernel':
                if zero_init and is_zero_init_kernel(name):
                    continue
                fan_in = shape[1] * shape[2] * shape[3] if len(shape) == 5 else shape[0]
                v = host[off: off + n]
                torch.nn.init.trunc_normal_(v, mean=0., std=1., a=-2., b=2., generator=g)
                v.mul_(math.sqrt(1.0 / fan_in) / 0.87962566103423978)
            elif leaf == 'scale':
                host[off: off + n] = 1.0
            elif leaf == 'bias':
                pass
            else:  # pos_emb, ref_pose_emb_*: normal(stddev=1/sqrt(D))  model/xunet.py:182-191
                host[off: off + n] = torch.randn(n, generator=g, device=gdev) / math.sqrt(POSE_EMB_DIM)
        return {'params': self.tree_from_flat(host.to(eng.device), S, B)}

    # ---- forward ------------------------------------------------------------------------------------------
    def apply(self, variables, batch, *, cond_mask, train: bool, rngs=None, rays=None) -> torch.Tensor:
        """XUNet.apply({'params': p}, batch, cond_mask=, train=, rngs={'dropout': key}) -> eps_hat (B,S,S,3), fp32, on device.
        rays (optional, also accepted as batch['rays']): precomputed (B,2,S,S,6) camera rays, see Engine.set_rays."""
        x = batch['x']
        B, S = int(x.shape[0]), int(x.shape[1])
        if tuple(np.shape(cond_mask)) != (B,):
            raise AssertionError(f'cond_mask.shape == (B,) violated: {np.shape(cond_mask)}')   # model/xunet.py:176
        eng = self.engine(B, S, False)
        flat = self.flat_from_tree(variables['params'], S, B)
        eng.load_inputs(batch, cond_mask=cond_mask)
        eng.set_rays(rays if rays is not None else batch.get('rays'))
        seed = _seed_of(rngs.get('dropout') if isinstance(rngs, dict) else rngs)
        try:
            return eng.forward(flat, train=train, seed=seed).clone()
        finally:
            eng.set_rays(None)

    # ---- vector-Jacobian products ------------------------------------------------------------------------
    def _train_forward(self, flat: torch.Tensor, batch, cond_mask, train: bool, rngs, rays):
        """The forward a VJP differentiates, on the training engine: (engine, eps_hat copy, the engine's forward count)."""
        x = batch['x']
        B, S = int(x.shape[0]), int(x.shape[1])
        if tuple(np.shape(cond_mask)) != (B,):
            raise AssertionError(f'cond_mask.shape == (B,) violated: {np.shape(cond_mask)}')   # model/xunet.py:176
        eng = self.engine(B, S, True)
        with torch.no_grad():
            eng.load_inputs({k: batch[k].detach() if isinstance(batch[k], torch.Tensor) else batch[k] for k in BATCH_KEYS},
                            cond_mask=cond_mask.detach() if isinstance(cond_mask, torch.Tensor) else cond_mask)
        rays = rays if rays is not None else batch.get('rays')
        eng.set_rays(rays.detach() if isinstance(rays, torch.Tensor) else rays)
        seed = _seed_of(rngs.get('dropout') if isinstance(rngs, dict) else rngs)
        try:
            eps = eng.forward(flat.detach(), train=train, seed=seed).clone()
        finally:
            eng.set_rays(None)
        return eng, eps, eng.forward_count

    @staticmethod
    def _check_current(eng: Engine, count: int):
        if eng.forward_count != count:
            raise RuntimeError(f'another forward ran on this engine since the one being differentiated (forward {count}, now '
                               f'{eng.forward_count}): its activations are gone; run the forward again')

    def vjp(self, variables, batch, *, cond_mask, train: bool, rngs=None, rays=None, camera_grads: bool = False):
        """jax.vjp over XUNet.apply: returns (eps_hat, vjp_fn).  vjp_fn(d_eps), d_eps = dL/d(eps_hat) a contiguous fp32 device
        tensor (B,S,S,3), returns (ParamTree of a copy of dL/dparams, {'x': dL/dx, 'z': dL/dz}); it may be called more than once,
        as long as no other forward has run on the training engine engine(B, S, True) in between (else RuntimeError).
        camera_grads=True adds the camera gradients to that dict: 'R1', 't1', 'R2', 't2', 'K' (R a free 3x3 matrix), or 'rays'
        (B,2,S,S,6) when explicit rays were given.  The log-SNR gets no gradient."""
        x = batch['x']
        B, S = int(x.shape[0]), int(x.shape[1])
        flat = self.flat_from_tree(variables['params'], S, B)
        explicit = (rays if rays is not None else batch.get('rays')) is not None
        eng, eps, count = self._train_forward(flat, batch, cond_mask, train, rngs, rays)

        def vjp_fn(d_eps):
            self._check_current(eng, count)
            if not camera_grads:
                grads, dx, dz = eng.backward_vjp(flat.detach(), d_eps, dx=True, dz=True)
                return self.tree_from_flat(grads.clone(), S, B, spec=eng.spec), {'x': dx.clone(), 'z': dz.clone()}
            grads, out = eng.backward_vjp_inputs(flat.detach(), d_eps, dx=True, dz=True, rays=explicit, cameras=not explicit)
            return self.tree_from_flat(grads.clone(), S, B, spec=eng.spec), {k: v.clone() for k, v in out.items()}

        return eps, vjp_fn

    def apply_autograd(self, flat_params: torch.Tensor, batch, *, cond_mask, train: bool, rngs=None, rays=None) -> torch.Tensor:
        """XUNet.apply as a torch.autograd.Function on the training engine: eps_hat (B,S,S,3) with a grad_fn, so that
        loss(eps_hat).backward() fills flat_params.grad and, for CUDA tensors batch['x'] / batch['z'] that require grad, their
        .grad.  Runs the same engine calls as vjp() (forward, then xunet_backward_vjp); the backward is once-differentiable and
        raises RuntimeError if another forward has run on the engine in between.
        Camera tensors batch['R1'], 't1', 'R2', 't2', 'K' (generated rays) or the explicit `rays` that are CUDA tensors requiring
        grad get their .grad too (xunet_backward_vjp_inputs, the same values as vjp(camera_grads=True)); the camera kernels run
        only when one of them needs a gradient.  The log-SNR gets no gradient."""
        rays = rays if rays is not None else batch.get('rays')
        cams = [batch[k] if isinstance(batch[k], torch.Tensor) else None for k in CAMERA_KEYS]
        ray_t = rays if isinstance(rays, torch.Tensor) else None
        return _XUNetVJP.apply(flat_params, batch['x'], batch['z'], *cams, ray_t, self, batch, cond_mask, train, rngs, rays)


class _XUNetVJP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flat_params, x, z, R1, t1, R2, t2, K, ray_t, model, batch, cond_mask, train, rngs, rays):
        eng, eps, count = model._train_forward(flat_params, dict(batch, x=x, z=z), cond_mask, train, rngs, rays)
        ctx.eng, ctx.count, ctx.explicit = eng, count, rays is not None
        ctx.cams = [(t.shape, t.dtype) if t is not None else None for t in (R1, t1, R2, t2, K, ray_t)]
        ctx.save_for_backward(flat_params)        # an in-place update of the parameters before backward() then raises
        return eps

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_eps):
        XUNet._check_current(ctx.eng, ctx.count)
        flat, = ctx.saved_tensors
        need_p, need_x, need_z = ctx.needs_input_grad[:3]
        need_cam = ctx.needs_input_grad[3:9]
        cameras = any(need_cam[:5]) and not ctx.explicit       # with explicit rays the cameras do not reach eps_hat
        rays = need_cam[5] and ctx.explicit
        d_eps = d_eps.to(torch.float32).contiguous()
        if not (cameras or rays):
            grads, dx, dz = ctx.eng.backward_vjp(flat.detach(), d_eps, dx=need_x, dz=need_z)
            return (grads.clone() if need_p else None, dx.clone() if need_x else None, dz.clone() if need_z else None,
                    None, None, None, None, None, None, None, None, None, None, None, None)
        grads, out = ctx.eng.backward_vjp_inputs(flat.detach(), d_eps, dx=need_x, dz=need_z, rays=rays, cameras=cameras)
        cam = []
        for key, need, meta in zip(CAMERA_KEYS + ('rays',), need_cam, ctx.cams):
            ok = need and key in out and (key == 'rays') == ctx.explicit
            cam.append(out[key].reshape(meta[0]).to(meta[1]).clone() if ok else None)
        return (grads.clone() if need_p else None, out['x'].clone() if need_x else None, out['z'].clone() if need_z else None,
                *cam, None, None, None, None, None, None)
