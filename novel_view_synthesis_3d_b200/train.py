"""Training step of the reference (train.py:36-76) on the CUDA path.

Reference call shapes are kept:
    state = create_train_state(rng, rng_dropout, learning_rate, train_batch_size, img_sidelength)
    loss, grads = apply_model(state, x, z, logsnr, R1, t1, R2, t2, K, noise)
    state = update_model(state, grads)
Differences by design (SURVEY Appendix C): the batch is SHARDED across ranks and gradients are averaged with one
NCCL all-reduce of the flat gradient bucket (the reference's pmap never calls pmean, train.py:49-76); cond_mask and the
dropout seed are fresh per step unless reference_quirks=True (the reference freezes both at trace time, train.py:64,66).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, replace
from typing import Optional

import numpy as np
import torch

from . import _lib
from . import dist as xdist
from .diffusion import diffusion_tables, min_snr_weights
from .distill import check_teacher, run_teacher
from .posthoc import PosthocEMA, check_posthoc_ema
from .sampling import check_prediction
from .xunet import XUNet, ParamTree, Engine, InputSlots, check_loss


@dataclass
class AdamState:
    """optax.adam(learning_rate) state (train.py:45): b1=.9, b2=.999, eps=1e-8."""
    mu: torch.Tensor
    nu: torch.Tensor
    count: int = 0


@dataclass
class Adam:
    """optax.adam hyper-parameters; with max_grad_norm / warmup_steps set, optax.chain(optax.clip_by_global_norm(max_grad_norm),
    optax.adam(optax.linear_schedule(0, learning_rate, warmup_steps)))."""
    learning_rate: float = 1e-4
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-8
    max_grad_norm: Optional[float] = None
    warmup_steps: int = 0

    @property
    def clip_or_warmup(self) -> bool:
        """The step clips the gradient or warms the learning rate up (and the state carries a ClipState)."""
        return self.max_grad_norm is not None or self.warmup_steps > 0


@dataclass
class ClipState:
    """Device block of gradient clipping and warm-up: the pre-clip global gradient norm of the last update, the scratch of
    its reduction kernel, and the number of updates skipped because that norm was not finite."""
    norm: torch.Tensor        # (1,) fp32
    scratch: torch.Tensor     # (GRAD_NORM_SCRATCH,) fp64
    skipped: torch.Tensor     # (1,) int64

    @staticmethod
    def zeros(device) -> "ClipState":
        return ClipState(norm=torch.zeros(1, dtype=torch.float32, device=device),
                         scratch=torch.zeros(_lib.GRAD_NORM_SCRATCH, dtype=torch.float64, device=device),
                         skipped=torch.zeros(1, dtype=torch.int64, device=device))


@dataclass
class TrainState:
    """Look-alike of flax.training.train_state.TrainState (fields used by train.py / sampling.py)."""
    step: int
    apply_fn: object
    params: ParamTree
    tx: Adam
    opt_state: AdamState
    model: XUNet = None
    batch_size: int = 0
    img_sidelength: int = 0
    grad_scale: float = 1.0
    reference_quirks: bool = False
    # exponential moving average of the weights (what DDPM-family models are sampled from), updated inside the Adam pass;
    # None when create_train_state(ema_decay=None)
    ema_params: Optional[ParamTree] = None
    ema_decay: Optional[float] = None
    # two power-function averages of the weights (post-hoc EMA, posthoc.py), updated inside the Adam pass; None unless
    # create_train_state(posthoc_ema=..)
    posthoc: Optional[PosthocEMA] = None
    # gradient-norm / skip-counter block; None unless create_train_state(max_grad_norm=..) or (warmup_steps=..)
    clip: Optional[ClipState] = None
    # training objective: 'frobenius' (the reference's ||eps_hat - noise||_F, train.py:67) or 'mse' (the mean squared error
    # of DDPM's L_simple, optionally weighted per sample); not part of the checkpoint
    loss: str = 'frobenius'
    # what the network is trained to predict: 'eps' (the noise) or 'v' (sqrt(abar) eps - sqrt(1 - abar) x0); recorded in
    # the checkpoint
    prediction: str = 'eps'
    # a progressively distilled student's {teacher_steps, rounds[, w]} (distill.Teacher.record), a consistency-distilled one's
    # {cd_steps[, w]} (distill.ConsistencyTeacher.record); None for any other model.  Recorded in the checkpoint
    distill: Optional[dict] = None
    _mask_rng: np.random.RandomState = None
    _frozen_mask: Optional[np.ndarray] = None

    def apply_gradients(self, *, grads, copy: bool = False) -> "TrainState":
        """TrainState.apply_gradients (train.py:76): one fused Adam pass over the flat buffers (plus the EMA update when the
        state carries one).

        Ownership: by default the flat parameter / moment / EMA buffers are updated IN PLACE and the returned state shares
        them, i.e. the OLD state's `params` alias the new values (the reference rebinds `state = update_model(state, ..)`
        and never looks at the old one, train.py:153).  copy=True gives the Flax contract literally: the old state keeps
        its values and the new state owns fresh buffers (3 x 4 bytes per parameter of extra traffic, 4 x 4 with EMA, 5 x 4
        with the two post-hoc averages).

        With clipping (tx.max_grad_norm) the global gradient norm is reduced first, into `clip.norm`; an update whose norm
        is not finite changes nothing but the counters and is counted in `skipped_steps`."""
        lib = _lib.load()
        flat_g = grads.flat if isinstance(grads, ParamTree) else grads
        S, B = self.img_sidelength, self.batch_size
        if copy:
            newp = self.model.tree_from_flat(self.params.flat.clone(), S, B)
            newe = None if self.ema_params is None else self.model.tree_from_flat(self.ema_params.flat.clone(), S, B)
            ph = self.posthoc
            newh = None if ph is None else replace(ph, a=self.model.tree_from_flat(ph.a.flat.clone(), S, B),
                                                   b=self.model.tree_from_flat(ph.b.flat.clone(), S, B))
            newc = None if self.clip is None else replace(self.clip, norm=self.clip.norm.clone(),
                                                          skipped=self.clip.skipped.clone())
            self = replace(self, params=newp, ema_params=newe, posthoc=newh, clip=newc,
                           opt_state=replace(self.opt_state, mu=self.opt_state.mu.clone(), nu=self.opt_state.nu.clone()))
        p = self.params.flat
        count = self.opt_state.count + 1
        st = torch.cuda.current_stream(p.device).cuda_stream
        _adam_launch(lib, self, flat_g, count, None, self.grad_scale, st)
        return replace(self, step=self.step + 1, opt_state=replace(self.opt_state, count=count))

    @property
    def skipped_steps(self) -> int:
        """Updates skipped because the gradient norm was not finite (reads the device counter: synchronises)."""
        return 0 if self.clip is None else int(self.clip.skipped.item())


def _adam_launch(lib, s: TrainState, flat_g: torch.Tensor, count: int, step_dev, grad_scale: float, stream: int) -> None:
    """One fused Adam pass over the flat buffers of `s`, with the EMA (or the two post-hoc averages), warm-up and clipping
    the state carries (the library runs plain Adam without the clip / warm-up prologue when there is neither).  With
    clipping the global-norm reduction runs first."""
    p, tx, c = s.params.flat, s.tx, s.clip
    ptr = lambda t: None if t is None else t.data_ptr()
    norm = None
    if tx.max_grad_norm is not None:
        _lib.check(lib.xunet_grad_global_norm(flat_g.data_ptr(), p.numel(), grad_scale, c.scratch.data_ptr(),
                                              c.norm.data_ptr(), stream), 'xunet_grad_global_norm')
        norm = c.norm
    skipped = None if c is None else c.skipped
    if s.posthoc is not None:
        ph = s.posthoc
        _lib.check(lib.xunet_adam_posthoc_step(p.data_ptr(), flat_g.data_ptr(), s.opt_state.mu.data_ptr(),
                                               s.opt_state.nu.data_ptr(), ph.a.flat.data_ptr(), ph.b.flat.data_ptr(),
                                               p.numel(), count, ptr(step_dev), tx.learning_rate, tx.b1, tx.b2, tx.eps,
                                               grad_scale, ph.gamma[0], ph.gamma[1], ptr(norm), tx.max_grad_norm or 0.0,
                                               tx.warmup_steps, ptr(skipped), stream), 'xunet_adam_posthoc_step')
        return
    ema = None if s.ema_params is None else s.ema_params.flat
    _lib.check(lib.xunet_adam_clip_step(p.data_ptr(), flat_g.data_ptr(), s.opt_state.mu.data_ptr(), s.opt_state.nu.data_ptr(),
                                        ptr(ema), p.numel(), count, ptr(step_dev), tx.learning_rate, tx.b1, tx.b2, tx.eps,
                                        grad_scale, s.ema_decay or 0.0, ptr(norm), tx.max_grad_norm or 0.0, tx.warmup_steps,
                                        ptr(skipped), stream), 'xunet_adam_clip_step')


def _opt_buffers(s: TrainState):
    """Every buffer one Adam pass writes that outlives the step (the flat buffers, and the skip counter)."""
    bufs = [s.params.flat, s.opt_state.mu, s.opt_state.nu]
    if s.ema_params is not None:
        bufs.append(s.ema_params.flat)
    if s.posthoc is not None:
        bufs += s.posthoc.flats()
    if s.clip is not None:
        bufs.append(s.clip.skipped)
    return bufs


def create_sample_data(batch_size, img_sidelength):
    """train.py:23-34."""
    r = np.random.random
    return dict(x=r((batch_size, img_sidelength, img_sidelength, 3)), z=r((batch_size, img_sidelength, img_sidelength, 3)),
                logsnr=r((batch_size,)), R1=r((batch_size, 3, 3)), t1=r((batch_size, 3)), R2=r((batch_size, 3, 3)),
                t2=r((batch_size, 3)), K=r((batch_size, 3, 3)), noise=r((batch_size, img_sidelength, img_sidelength, 3)))


def create_train_state(rng, rng_dropout, learning_rate, train_batch_size, img_sidelength, *, model: XUNet = None,
                       zero_init: bool = True, reference_quirks: bool = False, init_on_device: bool = False,
                       ema_decay: Optional[float] = None, max_grad_norm: Optional[float] = None,
                       warmup_steps: int = 0, loss: str = 'frobenius', prediction: str = 'eps',
                       posthoc_ema: Optional[tuple] = None) -> TrainState:
    """train.py:36-47.  Under torch.distributed the parameters of rank 0 are broadcast (the reference gives every
    device a different init, train.py:122-123 -- an ensemble, not data parallelism).

    ema_decay (e.g. 0.9999, Ho et al. 2020): keep `ema_params`, an exponential moving average of the weights updated in
    the same kernel as Adam, starting as a copy of the initial parameters.  Every rank updates its own copy; the parameters
    are identical across ranks after the all-reduce and Adam, so the copies stay identical without a collective.  None
    (default): no EMA buffer, the optimizer step is plain Adam.

    posthoc_ema (e.g. (0.05, 0.10), Karras et al. 2024): keep `posthoc`, two power-function averages of the weights of
    these relative widths sigma_rel (two different values in (0, 0.2887)), updated in the same kernel as Adam, from which
    posthoc.reconstruct rebuilds an EMA of any width after training out of the snapshots posthoc.save_snapshot writes.
    Both start as copies of the initial parameters, which the first update overwrites.  Every rank updates its own copies,
    identical across ranks like the EMA's.  Exclusive with ema_decay (ValueError).

    max_grad_norm (e.g. 1.0, Ho et al. 2020): clip the averaged gradient to this global L2 norm before Adam
    (optax.clip_by_global_norm).  The norm is reduced on the device in a fixed order, so runs stay bit-reproducible; an update
    whose norm is NaN or Inf is skipped entirely (the step count still advances) and counted in `state.skipped_steps`.
    warmup_steps (e.g. 5000): warm the learning rate up linearly from 0 over this many updates
    (optax.linear_schedule(0, learning_rate, warmup_steps)); 0 keeps it constant.  With the defaults (None, 0) the
    optimizer step is exactly the plain one.  Every rank computes the norm of the same all-reduced gradient, so the clip and
    skip decisions agree across ranks without a collective.

    loss: 'frobenius' (default) trains on the reference's ||eps_hat - noise||_F over the whole micro-batch.  'mse' trains on
    the mean squared error (1/B) sum_b w_b * mean_i (eps_hat - noise)_bi^2 of DDPM and 3DiM, whose per-sample weights w_b
    (all 1 unless a loss_weight is passed, e.g. from ForwardDiffusion(min_snr_gamma=..)) make per-sample weighting possible.
    With it, gradient accumulation and data parallelism give the gradient of the mean over the whole global batch.

    prediction: 'eps' (default) trains the network to predict the noise.  'v' trains it to predict
    v = sqrt(abar_t) eps - sqrt(1 - abar_t) x0 (Salimans & Ho 2022), from which x0 = sqrt(abar_t) z - sqrt(1 - abar_t) v
    loses at most the error of v (an eps error reaches x0 multiplied by sqrt(1/abar_t - 1), about 6e4 at t = 999).  It
    needs loss='mse'.  A TrainStep(data=..) then draws v targets on the device; the host-input calls (apply_model,
    TrainStep(batch, target)) take the v target (diffusion.v_target) where an eps state takes the noise.  Sample the
    result with Sampler(prediction='v')."""
    check_loss(loss)
    check_prediction(prediction)
    if prediction == 'v' and loss != 'mse':
        raise ValueError(f"prediction='v' needs loss='mse', got loss={loss!r}")
    if ema_decay is not None and not (0.0 <= ema_decay <= 1.0):
        raise ValueError(f'ema_decay must lie in [0, 1], got {ema_decay}')
    if posthoc_ema is not None:
        if ema_decay is not None:
            raise ValueError('ema_decay and posthoc_ema are exclusive: keep either a fixed-decay EMA or the two post-hoc '
                             'averages')
        posthoc_ema = check_posthoc_ema(posthoc_ema)
    if max_grad_norm is not None and not (float(max_grad_norm) > 0.0 and np.isfinite(float(max_grad_norm))):
        raise ValueError(f'max_grad_norm must be a finite number > 0, got {max_grad_norm}')
    if isinstance(warmup_steps, bool) or int(warmup_steps) != warmup_steps or warmup_steps < 0:
        raise ValueError(f'warmup_steps must be an integer >= 0, got {warmup_steps}')
    model = model or XUNet()
    sample = create_sample_data(train_batch_size, img_sidelength)
    params = model.init({'params': rng, 'dropout': rng_dropout}, sample, cond_mask=np.zeros(train_batch_size), train=True,
                        zero_init=zero_init, on_device=init_on_device)['params']
    world = xdist.world_size()
    xdist.broadcast_params(params.flat, src=0)
    opt = Adam(learning_rate, max_grad_norm=None if max_grad_norm is None else float(max_grad_norm),
               warmup_steps=int(warmup_steps))
    st = AdamState(mu=torch.zeros_like(params.flat), nu=torch.zeros_like(params.flat), count=0)
    mask_seed = int(np.asarray(rng_dropout).reshape(-1)[-1]) if rng_dropout is not None else 0
    # data parallel: every rank draws its OWN cond_mask stream (and dropout seeds, _dropout_seed) for its shard --
    # identical streams would drop sample b of every shard together, which is not a global batch of world*B
    mask_seed ^= (xdist.rank() * 0x9E3779B9) & 0x7FFFFFFF
    ema = None
    if ema_decay is not None:
        ema = model.tree_from_flat(params.flat.clone(), img_sidelength, train_batch_size)
    return TrainState(step=0, apply_fn=model.apply, params=params, tx=opt, opt_state=st, model=model,
                      batch_size=train_batch_size, img_sidelength=img_sidelength, grad_scale=1.0 / world,
                      reference_quirks=reference_quirks, ema_params=ema,
                      ema_decay=None if ema_decay is None else float(ema_decay),
                      posthoc=None if posthoc_ema is None else
                      PosthocEMA.create(model, params, posthoc_ema, img_sidelength, train_batch_size),
                      clip=ClipState.zeros(params.flat.device) if opt.clip_or_warmup else None, loss=loss,
                      prediction=prediction,
                      _mask_rng=np.random.RandomState(mask_seed & 0x7FFFFFFF))


def _dropout_seed(step_plus_1: int) -> int:
    """Dropout seed of optimisation step `step_plus_1` (1-based) on this rank: the rank sits in the high bits."""
    return (xdist.rank() << 40) + int(step_plus_1)


MAX_GRAD_ACCUM_STEPS = 256      # micro-batch indices must fit in bits 32-39 of the dropout seed (_micro_batch_seed)


def _micro_batch_seed(step_plus_1: int, j: int) -> int:
    """Dropout seed of micro-batch j of optimisation step `step_plus_1` under gradient accumulation: micro-batch 0 keeps
    _dropout_seed, micro-batch j adds j << 32.  j < 256 stays below the rank bits (40 and up), so every (rank, step, j) of a
    run below 2**32 steps has its own seed."""
    return _dropout_seed(step_plus_1) + (int(j) << 32)


def check_grad_accum_steps(k) -> int:
    """Validates TrainStep's grad_accum_steps: an int in [1, MAX_GRAD_ACCUM_STEPS]."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_GRAD_ACCUM_STEPS:
        raise ValueError(f'grad_accum_steps must be an integer in [1, {MAX_GRAD_ACCUM_STEPS}], got {k!r}')
    return int(k)


def check_accum_batch(batch: dict, noise, cond_mask, k: int, B: int, loss_weight=None) -> None:
    """Every array of a gradient-accumulation step (the batch dict, noise, and cond_mask and loss_weight when given) must
    have k*B rows: micro-batch j is rows [j*B, (j+1)*B).  Raises ValueError otherwise."""
    items = [(key, batch[key]) for key in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K')] + [('noise', noise)]
    if cond_mask is not None:
        items.append(('cond_mask', cond_mask))
    if loss_weight is not None:
        items.append(('loss_weight', loss_weight))
    for key, v in items:
        shape = tuple(v.shape) if hasattr(v, 'shape') else np.shape(v)
        rows = int(shape[0]) if shape else 0
        if rows != k * B:
            raise ValueError(f"{key} has leading dimension {rows}, expected grad_accum_steps * batch_size = {k} * {B} = {k * B}")


def check_loss_weight(loss: str, loss_weight, rows: int) -> None:
    """Per-sample loss weights: only with loss='mse', shape (rows,), and, when they are on the host, finite and >= 0 (device
    tensors are not read back).  Raises ValueError otherwise."""
    if loss_weight is None:
        return
    if loss != 'mse':
        raise ValueError(f"loss_weight needs a state built with loss='mse', this one uses loss={loss!r}")
    shape = tuple(loss_weight.shape) if hasattr(loss_weight, 'shape') else np.shape(loss_weight)
    if shape != (rows,):
        raise ValueError(f'loss_weight has shape {shape}, expected ({rows},)')
    if isinstance(loss_weight, torch.Tensor) and loss_weight.is_cuda:
        return
    w = loss_weight.detach().double().numpy() if isinstance(loss_weight, torch.Tensor) else np.asarray(loss_weight, np.float64)
    if not (np.isfinite(w).all() and (w >= 0).all()):
        raise ValueError('loss_weight must be finite and >= 0')


def _cond_mask(state: TrainState, B: int) -> np.ndarray:
    # train.py:64  np.where(np.random.random(B) > 0.1, 1, 0)
    if state.reference_quirks:
        if state._frozen_mask is None:
            state._frozen_mask = np.where(state._mask_rng.random_sample(B) > 0.1, 1, 0).astype(np.float32)
        return state._frozen_mask
    return np.where(state._mask_rng.random_sample(B) > 0.1, 1, 0).astype(np.float32)


def apply_model(state: TrainState, batch_x, batch_z, batch_logsnr, batch_R1, batch_t1, batch_R2, batch_t2, batch_K,
                batch_noise, *, cond_mask=None, loss_weight=None):
    """train.py:49-72: forward with train=True, the state's loss (||eps_hat - noise||_F by default), gradients w.r.t. all
    parameters.  batch_noise is the regression target: the noise of z for a state built with prediction='eps', the v target
    (diffusion.v_target of the clean target view, that noise and the timestep) for prediction='v'.  loss_weight: per-sample
    weights (B,) of loss='mse', host or device (all 1 when None).
    Returns (loss: 0-d device tensor, grads: ParamTree view of the flat gradient bucket).  With
    torch.distributed initialised the gradient bucket is all-reduced (sum) here; update_model applies 1/world."""
    B, S = int(batch_x.shape[0]), int(batch_x.shape[1])
    check_loss_weight(state.loss, loss_weight, B)
    eng = state.model.engine(B, S, True)
    batch = dict(x=batch_x, z=batch_z, logsnr=batch_logsnr, R1=batch_R1, t1=batch_t1, R2=batch_R2, t2=batch_t2, K=batch_K)
    mask = _cond_mask(state, B) if cond_mask is None else cond_mask
    eng.load_inputs(batch, cond_mask=mask, noise=batch_noise, loss_weight=loss_weight)
    seed = 0 if state.reference_quirks else _dropout_seed(state.step + 1)   # PRNGKey(0) frozen at trace time, train.py:66
    eng.forward(state.params.flat, train=True, seed=seed)
    loss, grads = eng.backward(state.params.flat, loss=state.loss,
                               loss_weight=None if loss_weight is None else eng.inp['loss_weight'])
    xdist.allreduce_sum_(grads, bucket_elems=64 << 20)
    # the loss is a copy; `grads` are views of the engine's gradient bucket (valid until the next backward of this plan)
    return loss[0].clone(), state.model.tree_from_flat(grads, S, B)


def update_model(state: TrainState, grads) -> TrainState:
    """train.py:74-76."""
    return state.apply_gradients(grads=grads)


class TrainStep:
    """The fused production step: pinned H2D staging -> forward -> backward (gradient buckets all-reduced over NCCL as they
    become final, overlapping the rest of the backward) -> Adam with 1/world folded in.  Semantically apply_model +
    update_model (train.py:142-153).

    Execution modes (chosen at the first call):
      world == 1                : CUDA graph [forward + backward + Adam]
      world > 1, NCCL           : ONE CUDA graph [forward + backward + bucketed all-reduces + Adam]; the collectives are
                                  captured on NCCL's stream as parallel branches of the graph
      world > 1, other backends : graph [forward + backward]; eager bucketed all-reduce; graph [Adam]   (gloo in tests, or
                                  NCCL when capturing the collectives fails)
      use_graph=False           : everything eager; the bucket hook still overlaps the all-reduces with the backward

    With gradient clipping the global-norm reduction runs right before Adam in every mode (after the all-reduce), inside
    the same graph as Adam.

    grad_accum_steps=k (optax.MultiSteps(.., every_k_schedule=k)): each call takes k*B samples per rank (B =
    state.batch_size) and runs k forward/backward passes of B samples, micro-batch j being rows [j*B, (j+1)*B); the first
    backward overwrites the flat gradient buffer, the others add into it (xunet_backward_accumulate), and one update (norm,
    Adam, EMA or post-hoc averages) follows with grad_scale = 1/(world*k): Adam of the mean micro-batch gradient.  The loss of each micro-batch is
    its own Frobenius norm, so this is not the gradient of one batch of k*B samples (as data parallelism is not).  Under
    data parallelism only the last backward carries the bucket hook, so the all-reduce covers the whole sum.  The returned
    loss is the mean of the k micro-batch losses; `step` and the Adam count advance by one per call.  k = 1 (the default)
    runs exactly the step without accumulation.  With a state built with loss='mse' every micro-batch holds B samples of the
    same mean, so the update is that of the mean squared error over all world*k*B samples, and the returned loss is that
    mean; per-sample weights, when given, have k*B rows like cond_mask and are staged with the batch.

    A captured graph holds the NCCL kernels of the process group it was captured with: drop the TrainStep (or call
    `release_graphs()`) before `torch.distributed.destroy_process_group()`.

    data=DeviceScenes (srn_data): the step draws its own batches from the views held in device memory and is called with no
    arguments, `loss = step()`.  Each micro-batch's forward is preceded by one kernel (xunet_srn_batch) that draws the B
    (source, target) pairs, gathers their pixels and poses and runs the forward diffusion with p_uncond (and, with
    min_snr_gamma, a state built with loss='mse' gets the min-SNR-gamma weights of the drawn timesteps), all in the graph:
    no host work and no host->device copy per step (`h2d_bytes` is 0; the host cond_mask stream is not used).  The draw is a
    function of (data_seed, Adam count, micro-batch, rank): sample b of micro-batch j on rank r of the update at Adam count c
    has the draw index g = ((c k + j) world + r) B + b, so the ranks and micro-batches of one update partition a global batch
    of world k B draws (the host loader instead gives every rank its own stream), and each run of N consecutive draws visits
    every view once as the source, in a keyed random order that changes every such epoch.  Epochs are not aligned with
    updates: an update may take its first draws from one epoch and the rest from the next (nothing is dropped).  Since the
    order follows the Adam count, restore_train_state + the same store and data_seed continue the data stream exactly.
    For a state built with prediction='v' the same kernel (xunet_srn_batch_v) writes the v target of each draw where an
    eps state gets its noise, and min_snr_gamma gives the v weights; nothing else in the step changes.

    teacher=distill.Teacher (with data=): progressive distillation of the teacher into this state, a v / mse student
    (distill.create_distill_state).  Per micro-batch, before the student's forward and backward, the step draws the batch
    with t on the student grid (xunet_srn_batch_distill, cond_mask 1), runs the teacher forward, its first DDIM step, the
    second teacher forward (static conditioning on: the same poses, K, mask and parameters) and the target kernel, which
    writes the v target of the teacher's two steps into the slot's regression target.  Everything else -- accumulation,
    clipping, warm-up, EMA, data parallelism and the single-graph capture -- is the data= step's.  Raises ValueError without
    data=, for a state that is not prediction='v' with loss='mse', with reference_quirks or min_snr_gamma, for an odd teacher
    grid, and when the teacher's S, B, device or model configuration differ from the state's.

    teacher=distill.ConsistencyTeacher (with data=): consistency distillation, with the same checks (but any grid of N >= 2).
    Per micro-batch the step draws t on the teacher grid, runs the teacher forward and its DDIM step (xunet_cd_teacher_step),
    then the target forward -- this state's own parameters, train=0, on its training engine, at the stepped z -- and the
    target kernel (xunet_cd_target), which writes v* into the slot's regression target; the student's forward and backward
    follow as above.
    """

    def __init__(self, state: TrainState, *, use_graph: bool = True, bucket_mb: float = 128.0, allreduce: bool = True,
                 grad_accum_steps: int = 1, data=None, data_seed: int = 0, p_uncond: float = 0.1,
                 min_snr_gamma: Optional[float] = None, teacher=None):
        self.k = check_grad_accum_steps(grad_accum_steps)
        self.data = data
        self.teacher = teacher
        if teacher is not None:
            check_teacher(state, teacher, data)
            if min_snr_gamma is not None:
                raise ValueError('a distilled student is trained with the plain mse (SNR + 1 weighting of v): no min_snr_gamma')
        if data is None:
            if min_snr_gamma is not None:
                raise ValueError('min_snr_gamma weights the batches a data= step draws; without data= pass loss_weight')
        else:
            if state.reference_quirks:
                raise ValueError('data= draws a fresh cond_mask for every sample; reference_quirks=True freezes it')
            if min_snr_gamma is not None and state.loss != 'mse':
                raise ValueError(f"min_snr_gamma needs a state built with loss='mse', this one uses loss={state.loss!r}")
            if data.S != state.img_sidelength:
                raise ValueError(f'the store holds views at S = {data.S}, the state trains at S = {state.img_sidelength}')
        self.state = state
        self.mse = state.loss == 'mse'      # the captured graph reads each slot's loss weights in place
        self.eng: Engine = state.model.engine(state.batch_size, state.img_sidelength, True)
        self.dev = self.eng.device
        # the k micro-batches' inputs, dropout seeds and losses, all in device memory: the k forward/backward pairs of one
        # graph read them in place, and a replay sees the seeds advance.  k = 1: the engine's own buffers, and `loss` is the
        # engine's loss slot rather than a mean of one
        if self.k == 1:
            self.inputs, self.seeds, self.losses = self.eng.inputs, self.eng.seed, self.eng.loss
            self.loss = self.eng.loss
        else:
            self.inputs = InputSlots(self.eng.B, self.eng.S, self.k, self.dev)
            self.seeds = torch.zeros(self.k, dtype=torch.int64, device=self.dev)
            self.losses = torch.zeros(self.k, dtype=torch.float32, device=self.dev)
            self.loss = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self._hook = False
        self.lib = _lib.load()
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.world = xdist.world_size()
        self.use_graph = use_graph
        self.graph_fb = None      # forward+backward (+ all-reduce + adam when everything is in one graph)
        self.graph_opt = None     # adam (two-graph mode only)
        self.stream = torch.cuda.Stream(device=self.dev) if use_graph else None
        self.allreduce = allreduce and self.world > 1       # allreduce=False: measurement knob (compute-only step at N>1)
        self.bucket_bytes = int(bucket_mb * (1 << 20))
        self.reducer = xdist.GradReducer(self.eng.grads) if self.world > 1 else None
        if self.reducer is not None:
            self.reducer.enabled = self.allreduce
        backend = torch.distributed.get_backend() if self.world > 1 else None
        self.capture_collectives = self.world > 1 and backend == 'nccl' and use_graph
        self.mode = None
        self._synced_count = None
        self._sync_counters()
        if data is not None:
            if data.device != self.dev:
                raise ValueError(f'the store lives on {data.device}, the state trains on {self.dev}')
            self.data_seed = int(data_seed) & 0xFFFFFFFFFFFFFFFF
            self.p_uncond = float(p_uncond)
            sqrt_ac, sqrt_1mac = diffusion_tables()
            self.sqrt_ac = torch.as_tensor(sqrt_ac).to(self.dev)
            self.sqrt_1mac = torch.as_tensor(sqrt_1mac).to(self.dev)
            self.snr_weight = None if min_snr_gamma is None else \
                torch.as_tensor(min_snr_weights(min_snr_gamma, prediction=state.prediction), dtype=torch.float32).to(self.dev)
            self.h2d_bytes = 0

    @property
    def grad_norm(self) -> Optional[torch.Tensor]:
        """Global L2 norm of the averaged gradient of the step just run, before clipping: a 0-d device view (read or copy
        it before the next step).  None unless the state clips (create_train_state(max_grad_norm=..))."""
        s = self.state
        return None if s.tx.max_grad_norm is None else s.clip.norm[0]

    def release_graphs(self):
        self.graph_fb = self.graph_opt = None

    def _sync_counters(self):
        """Adam step counter and dropout seed live on the device (a replayed graph sees them advance); re-derive them from
        the host-side state whenever something else (apply_model / update_model, a restored checkpoint) moved it."""
        s = self.state
        if self._synced_count != s.opt_state.count:
            self.step_dev.fill_(s.opt_state.count)
            seeds = [0 if s.reference_quirks else _micro_batch_seed(s.opt_state.count, j) for j in range(self.k)]
            self.seeds.copy_(torch.tensor(seeds, dtype=torch.int64))
            self._synced_count = s.opt_state.count

    def _draw(self, j: int):
        """Micro-batch j of the current update, drawn from the device store into input slot j (xunet_srn_batch, or
        xunet_srn_batch_v with the v target in the slot's noise segment)."""
        d, inp = self.data, self.inputs.inp[j]
        ptr = lambda t: None if t is None else t.data_ptr()
        st = torch.cuda.current_stream(self.dev).cuda_stream
        head = (C.byref(d.c_store), self.step_dev.data_ptr(), self.data_seed, j, self.k, xdist.rank(), self.world, self.eng.B,
                self.sqrt_ac.data_ptr(), self.sqrt_1mac.data_ptr(), self.p_uncond, ptr(self.snr_weight),
                C.byref(self.inputs.cbatch[j]))
        tail = (inp['loss_weight'].data_ptr() if self.mse else None, None, None, st)
        if self.state.prediction == 'v':
            _lib.check(self.lib.xunet_srn_batch_v(*head, None, inp['noise'].data_ptr(), *tail), 'xunet_srn_batch_v')
        else:
            _lib.check(self.lib.xunet_srn_batch(*head, inp['noise'].data_ptr(), *tail), 'xunet_srn_batch')

    def _fwd_bwd(self):
        e, s = self.eng, self.state
        if not s.reference_quirks:
            self.seeds.add_(1)
        self.step_dev.add_(1)
        hook = self._hook
        try:
            if hook:
                self._set_hook(False)        # a bucket is final only in the last backward
            for j in range(self.k):
                last = j == self.k - 1
                sd = self.seeds[j:j + 1]
                if self.teacher is not None:
                    run_teacher(self, j)
                elif self.data is not None:
                    self._draw(j)
                e.forward(s.params.flat, train=True, inputs=(self.inputs, j), seed_dev=sd)
                if last:
                    self._set_hook(hook)
                    if self.reducer is not None:
                        self.reducer.begin()
                e.backward(s.params.flat, accumulate=j > 0, inputs=(self.inputs, j), seed_dev=sd,
                           loss_out=self.losses[j:j + 1], loss=s.loss,
                           loss_weight=self.inputs.inp[j]['loss_weight'] if self.mse else None)
        finally:
            self._set_hook(hook)
        if self.k > 1:
            torch.mean(self.losses, 0, keepdim=True, out=self.loss)

    def _adam(self):
        st = torch.cuda.current_stream(self.dev).cuda_stream
        _adam_launch(self.lib, self.state, self.eng.grads, 0, self.step_dev, 1.0 / (self.world * self.k), st)

    def _full_step(self):
        self._fwd_bwd()
        if self.reducer is not None:
            self.reducer.wait()
        self._adam()

    def _set_hook(self, on: bool):
        self._hook = on
        if self.reducer is None:
            return
        self.eng.set_bucket_callback(self.reducer.on_bucket if on else None, self.bucket_bytes)

    def _capture(self):
        one_graph = self.world == 1 or self.capture_collectives
        # warm-up and capture advance the seeds and the step counter and, with Adam in the graph, run real updates: snapshot
        # what they write and restore it afterwards.  The synchronize orders the snapshot before the warm-up's stream.
        saved = [self.seeds, self.step_dev] + (_opt_buffers(self.state) if one_graph else [])
        backup = [t.clone() for t in saved]
        torch.cuda.synchronize(self.dev)
        retry = False
        try:
            with torch.cuda.stream(self.stream):
                self._set_hook(one_graph)
                if one_graph:
                    self._full_step()                    # warm-up outside capture (also initialises the NCCL communicator)
                else:
                    self._fwd_bwd()
                self.stream.synchronize()
                self.graph_fb = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_fb, stream=self.stream):
                    if one_graph:
                        self._full_step()
                    else:
                        self._fwd_bwd()
                if not one_graph:
                    self.graph_opt = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(self.graph_opt, stream=self.stream):
                        self._adam()
            self.mode = 'one_graph' if one_graph else 'two_graphs_eager_collectives'
        except Exception:
            if not (one_graph and self.world > 1):
                raise
            # capturing the collectives failed: fall back to eager all-reduces between two graphs
            self.capture_collectives = False
            self.graph_fb = self.graph_opt = None
            retry = True
        finally:
            self._set_hook(False)
        torch.cuda.synchronize(self.dev)
        for t, b in zip(saved, backup):
            t.copy_(b)
        if retry:
            self._capture()

    def __call__(self, batch: Optional[dict] = None, noise=None, cond_mask=None, loss_weight=None) -> torch.Tensor:
        """One optimisation step on host (or device) inputs; returns the loss as a 0-d device tensor (a view of the step's
        loss slot: read or copy it before the next step).  `noise` is the regression target: the noise for a state built
        with prediction='eps', the v target (diffusion.v_target) for prediction='v'.  With grad_accum_steps=k every array has k*B rows, and the loss
        is the mean of the k micro-batch losses.  loss_weight: per-sample weights of a loss='mse' state (all 1 when None).
        A step built with data= draws its own batches and takes no arguments."""
        s = self.state
        if self.data is not None:
            if batch is not None or noise is not None or cond_mask is not None or loss_weight is not None:
                raise ValueError('this TrainStep draws its batches from its data= store: call it with no arguments')
            self._sync_counters()
        else:
            if batch is None or noise is None:
                raise TypeError('TrainStep() without data= needs a batch and its noise')
            if self.k > 1:
                check_accum_batch(batch, noise, cond_mask, self.k, self.eng.B, loss_weight)
            check_loss_weight(s.loss, loss_weight, self.k * self.eng.B)
            if self.mse and loss_weight is None:
                loss_weight = np.ones(self.k * self.eng.B, np.float32)    # the slots may still hold the last call's weights
            self._sync_counters()
            # micro-batch j draws the j-th B values of the rank's cond_mask stream
            mask = np.concatenate([_cond_mask(s, self.eng.B) for _ in range(self.k)]) if cond_mask is None else cond_mask
            self.h2d_bytes = self.inputs.load(batch, cond_mask=mask, noise=noise, loss_weight=loss_weight)
        if self.use_graph:
            if self.graph_fb is None:
                self._capture()
            self.graph_fb.replay()
            if self.graph_opt is not None:
                if self.allreduce:
                    xdist.allreduce_sum_(self.eng.grads, bucket_elems=self.bucket_bytes // 4)
                self.graph_opt.replay()
        else:
            self.mode = 'eager'
            self._set_hook(True)
            try:
                self._full_step()
            finally:
                self._set_hook(False)
        s.step += 1
        s.opt_state.count += 1
        self._synced_count = s.opt_state.count
        return self.loss[0]
