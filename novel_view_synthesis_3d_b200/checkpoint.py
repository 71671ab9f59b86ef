"""Flax checkpoint import / export for the X-UNet parameter tree  (SURVEY 8(f) row 1).

The reference saves `train_state.params` with `flax.training.checkpoints.save_checkpoint(ckpt_dir, target, step,
prefix='model', overwrite=True)` (train.py:159-167) -- every leaf carries a leading per-device axis because the state is
pmapped -- and restores it in sampling.py:106-114.  Flax (0.6.4) is not installable here, so this module restates its
published on-disk format (flax/serialization.py): a msgpack map of the nested state dict whose ndarray leaves are msgpack
ExtType(code=1) payloads = msgpack-packed `(shape, dtype_name, raw C-order bytes)`; numpy scalars are ExtType(3);
arrays larger than 2**30 bytes are stored as a dict of chunks {'__msgpack_chunked_array__': True, 'shape': {'0':..}, 'chunks': {'0':..}}.
File name: f'{prefix}{step}' inside ckpt_dir.

save_train_state / restore_train_state extend this to the whole training state (parameters, Adam moments and count, step,
the weight EMA or the two post-hoc averages, and the host cond_mask streams), so a run can be resumed where it stopped.
"""
from __future__ import annotations

import os
import re
import warnings
from typing import Dict, Optional

import msgpack
import numpy as np

from .xunet import _nest, pack_flat

_EXT_NDARRAY, _EXT_NATIVE_COMPLEX, _EXT_NPSCALAR = 1, 2, 3
_MAX_CHUNK = 2 ** 30


def _ndarray_to_bytes(arr: np.ndarray) -> bytes:
    arr = np.asarray(arr)
    return msgpack.packb((arr.shape, arr.dtype.name, arr.tobytes('C')), use_bin_type=True)


def _ndarray_from_bytes(data: bytes) -> np.ndarray:
    shape, dtype_name, buf = msgpack.unpackb(data, raw=False)
    return np.frombuffer(buf, dtype=np.dtype(dtype_name)).reshape(shape).copy()


def _ext_pack(x):
    if isinstance(x, np.ndarray):
        return msgpack.ExtType(_EXT_NDARRAY, _ndarray_to_bytes(x))
    if isinstance(x, np.generic):
        return msgpack.ExtType(_EXT_NPSCALAR, _ndarray_to_bytes(np.asarray(x)))
    if isinstance(x, complex):
        return msgpack.ExtType(_EXT_NATIVE_COMPLEX, msgpack.packb((x.real, x.imag)))
    return x


def _ext_unpack(code, data):
    if code == _EXT_NDARRAY:
        return _ndarray_from_bytes(data)
    if code == _EXT_NPSCALAR:
        return _ndarray_from_bytes(data)[()]
    if code == _EXT_NATIVE_COMPLEX:
        re_, im_ = msgpack.unpackb(data)
        return complex(re_, im_)
    return msgpack.ExtType(code, data)


def _chunk(tree):
    if isinstance(tree, dict):
        return {k: _chunk(v) for k, v in tree.items()}
    if isinstance(tree, np.ndarray) and tree.size * tree.dtype.itemsize > _MAX_CHUNK:
        flat = tree.reshape(-1)
        per = max(1, _MAX_CHUNK // tree.dtype.itemsize)
        chunks = [flat[i:i + per] for i in range(0, flat.size, per)]
        # flax stores tuples as {'0': .., '1': ..} dicts (msgpack strict_types)
        return {'__msgpack_chunked_array__': True, 'shape': {str(i): int(v) for i, v in enumerate(tree.shape)},
                'chunks': {str(i): c for i, c in enumerate(chunks)}}
    return tree


def _unchunk(tree):
    if isinstance(tree, dict):
        if tree.get('__msgpack_chunked_array__'):
            chunks = tree['chunks']
            parts = [chunks[str(i)] for i in range(len(chunks))]
            shp = tree['shape']
            shape = tuple(shp[str(i)] for i in range(len(shp))) if isinstance(shp, dict) else tuple(shp)
            return np.concatenate([np.asarray(p).reshape(-1) for p in parts]).reshape(shape)
        return {k: _unchunk(v) for k, v in tree.items()}
    return tree


def msgpack_serialize(tree: dict) -> bytes:
    """flax.serialization.msgpack_serialize for nested dicts of numpy arrays."""
    def to_np(t):
        if isinstance(t, dict):
            return {str(k): to_np(v) for k, v in t.items()}
        if hasattr(t, 'detach'):          # torch tensor
            return t.detach().cpu().numpy()
        return np.asarray(t) if not isinstance(t, (int, float, str, bool)) else t
    return msgpack.packb(_chunk(to_np(tree)), default=_ext_pack, strict_types=True, use_bin_type=True)


def msgpack_restore(data: bytes) -> dict:
    """flax.serialization.msgpack_restore."""
    return _unchunk(msgpack.unpackb(data, ext_hook=_ext_unpack, raw=False, strict_map_key=False))


def strip_device_axis(tree: dict, device_index: int = 0) -> dict:
    """The reference checkpoints pmapped params: every leaf is (n_devices, ...) (train.py:161-167). Take one replica."""
    if isinstance(tree, dict):
        return {k: strip_device_axis(v, device_index) for k, v in tree.items()}
    return np.asarray(tree)[device_index]


def save_checkpoint(ckpt_dir: str, target, step: int, prefix: str = 'model', overwrite: bool = True,
                    add_device_axis: bool = False) -> str:
    """checkpoints.save_checkpoint look-alike (train.py:161-167).  `target` = nested param dict (ParamTree / numpy / torch)."""
    os.makedirs(ckpt_dir, exist_ok=True)
    path = os.path.join(ckpt_dir, f'{prefix}{step}')
    if os.path.exists(path) and not overwrite:
        raise FileExistsError(path)
    tree = target
    if add_device_axis:
        def add(t):
            if isinstance(t, dict):
                return {k: add(v) for k, v in t.items()}
            a = t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)
            return a[None]
        tree = add(target)
    if overwrite:   # flax removes older checkpoints with the same prefix when overwrite=True
        for f in os.listdir(ckpt_dir):
            if re.fullmatch(re.escape(prefix) + r'\d+', f) and f != os.path.basename(path):
                os.remove(os.path.join(ckpt_dir, f))
    tmp = path + '.tmp'
    with open(tmp, 'wb') as fh:
        fh.write(msgpack_serialize(tree))
    os.replace(tmp, path)
    return path


def latest_checkpoint(ckpt_dir: str, prefix: str = 'model') -> Optional[str]:
    best, best_step = None, -1
    if not os.path.isdir(ckpt_dir):
        return None
    for f in os.listdir(ckpt_dir):
        # flax globs f'{prefix}*' and sorts naturally: 'model0' is found both by prefix 'model' (step 0) and by prefix
        # 'model0' (sampling.py:109), where nothing follows the prefix
        m = re.fullmatch(re.escape(prefix) + r'(\d*)', f)
        if m:
            step = int(m.group(1)) if m.group(1) else 0
            if step > best_step:
                best, best_step = os.path.join(ckpt_dir, f), step
    return best


def restore_checkpoint(ckpt_dir: str, prefix: str = 'model', device_index: Optional[int] = None) -> Optional[dict]:
    """checkpoints.restore_checkpoint look-alike (sampling.py:106-110): returns the nested param dict of the latest
    f'{prefix}<step>' file, or None if there is none (the reference raises FileNotFoundError in that case, :111-112).
    If the leaves carry the pmap device axis (auto-detected on GroupNorm scales: 2-D instead of 1-D) one replica is taken."""
    path = ckpt_dir if os.path.isfile(ckpt_dir) else latest_checkpoint(ckpt_dir, prefix)
    if path is None:
        return None
    with open(path, 'rb') as fh:
        tree = msgpack_restore(fh.read())
    if 'params' in tree and isinstance(tree['params'], dict) and 'Conv_0' not in tree:
        tree = tree['params']      # a whole TrainState was saved
    probe = tree.get('GroupNorm_0', {}).get('GroupNorm_0', {}).get('scale')
    has_axis = probe is not None and np.asarray(probe).ndim == 2
    if device_index is not None or has_axis:
        tree = strip_device_axis(tree, device_index or 0)
    return tree


# ---- resumable training state ------------------------------------------------------------------------------------------
# The tree is built and parsed by pure functions over numpy arrays (train_state_tree / parse_train_state_tree), so its
# layout can be checked without a GPU; save_train_state / restore_train_state move the device buffers in and out.

def leaf_tree(flat: np.ndarray, spec) -> dict:
    """Flat host buffer -> nested {leaf: array} in the Flax tree shape; spec = {name: (shape, offset)} (ParamTree.spec)."""
    return _nest({name: flat[off: off + int(np.prod(shape))].reshape(shape) for name, (shape, off) in spec.items()})


def rng_state_dict(rng: np.random.RandomState, frozen_mask: Optional[np.ndarray] = None) -> dict:
    """One rank's host cond_mask stream (TrainState._mask_rng, and _frozen_mask under reference_quirks)."""
    kind, keys, pos, has_gauss, cached = rng.get_state()
    d = {'keys': np.asarray(keys, dtype=np.uint32), 'pos': int(pos), 'has_gauss': int(has_gauss),
         'cached_gaussian': float(cached)}
    if frozen_mask is not None:
        d['frozen_mask'] = np.asarray(frozen_mask, dtype=np.float32)
    return d


def _set_rng_state(rng: np.random.RandomState, d: dict):
    rng.set_state(('MT19937', np.asarray(d['keys'], dtype=np.uint32), int(d['pos']), int(d['has_gauss']),
                   float(d['cached_gaussian'])))
    return np.asarray(d['frozen_mask'], dtype=np.float32) if 'frozen_mask' in d else None


def train_state_tree(params: dict, mu: dict, nu: dict, count: int, step: int, *, ema: Optional[dict] = None,
                     rng: Optional[list] = None, add_device_axis: bool = False, clip: bool = False,
                     schedule: bool = False, skipped: Optional[int] = None, prediction: Optional[str] = None,
                     distill: Optional[dict] = None, posthoc: Optional[tuple] = None,
                     posthoc_sigma_rel: Optional[tuple] = None) -> dict:
    """The nested dict flax.serialization.to_state_dict gives for a flax.training.train_state.TrainState with
    tx=optax.adam(lr), i.e. chain(scale_by_adam, scale(-lr)):

        {'step': int32, 'params': {...}, 'opt_state': {'0': {'count': int32, 'mu': {...}, 'nu': {...}}, '1': {}}}

    With gradient clipping (clip=True) and / or a learning-rate schedule (schedule=True) the optimizer is
    optax.chain(optax.clip_by_global_norm(c), optax.adam(schedule)); clip_by_global_norm keeps an empty state and
    scale_by_schedule keeps its own count, so 'opt_state' becomes

        clip and schedule: {'0': {}, '1': {'0': {'count', 'mu', 'nu'}, '1': {'count': int32}}}
        clip only:         {'0': {}, '1': {'0': {'count', 'mu', 'nu'}, '1': {}}}
        schedule only:     {'0': {'count', 'mu', 'nu'}, '1': {'count': int32}}

    (the schedule's count equals Adam's: both advance once per update).  Plus 'ema_params' (a params-shaped tree) when an
    EMA is kept, 'rng': {'<rank>': rng_state_dict(..)} for the host cond_mask stream of every rank, and 'skipped_steps'
    (int64, updates skipped for a non-finite gradient norm) and 'prediction' (the string 'eps' or 'v': what the network was
    trained to predict) when given, and 'distill' ({'teacher_steps', 'rounds'[, 'w']}, a progressively distilled student's
    record) when given, and 'posthoc_ema': {'0': tree, '1': tree} with 'posthoc_sigma_rel' (fp64, both widths) for the two
    post-hoc averages (posthoc = (a, b), params-shaped trees) when given.  The Flax / optax layouts are restated from memory
    of their published sources and have not been checked against files written by the packages themselves.
    add_device_axis=True gives every Flax leaf (not 'rng' / 'skipped_steps') the leading pmap axis of length 1, as the
    reference's pmapped state carries it (train.py:161-167).  params / mu / nu / ema: nested dicts of numpy arrays
    (leaf_tree)."""
    def ax(t):
        if isinstance(t, dict):
            return {k: ax(v) for k, v in t.items()}
        return np.asarray(t)[None] if add_device_axis else np.asarray(t)
    adam = {'count': np.asarray(count, dtype=np.int32), 'mu': mu, 'nu': nu}
    sched = {'count': np.asarray(count, dtype=np.int32)} if schedule else {}
    opt = {'0': {}, '1': {'0': adam, '1': sched}} if clip else {'0': adam, '1': sched}
    tree = {'step': np.asarray(step, dtype=np.int32), 'params': params, 'opt_state': opt}
    if ema is not None:
        tree['ema_params'] = ema
    if posthoc is not None:
        tree['posthoc_ema'] = {'0': posthoc[0], '1': posthoc[1]}
    tree = ax(tree)
    if posthoc is not None:
        tree['posthoc_sigma_rel'] = np.asarray(posthoc_sigma_rel, dtype=np.float64)
    if rng is not None:
        tree['rng'] = {str(r): d for r, d in enumerate(rng)}
    if skipped is not None:
        tree['skipped_steps'] = np.asarray(skipped, dtype=np.int64)
    if prediction is not None:
        tree['prediction'] = str(prediction)
    if distill is not None:
        tree['distill'] = {k: (float(v) if k == 'w' else int(v)) for k, v in distill.items()}
    return tree


def parse_train_state_tree(tree: dict, spec, nparams: int) -> dict:
    """Inverse of train_state_tree onto flat fp32 host buffers laid out by `spec`.  Returns {'step', 'count', 'params',
    'mu', 'nu', 'ema' (None if the file has none), 'rng' (list indexed by rank, or None), 'skipped' (0 if the file has
    none), 'prediction' ('eps' if the file has none: files written before v-prediction existed hold eps models), 'distill'
    (None if the file has none: a model that is not a distilled student), 'posthoc' ((a, b) flat buffers, None if the file
    has none) and 'posthoc_sigma_rel' (a tuple, None if the file has none)}.  Accepts all four optimizer layouts (with and without clipping, with and without a schedule), so a run may
    turn either on or off when it resumes; a schedule count that differs from Adam's raises ValueError.  Detects the pmap
    device axis from the shape of 'step' and takes replica 0.  Missing / unexpected leaves raise KeyError, wrong shapes
    ValueError."""
    tree = dict(tree)
    rng = tree.pop('rng', None)
    skipped = tree.pop('skipped_steps', None)
    prediction = str(tree.pop('prediction', 'eps'))
    distill = tree.pop('distill', None)
    ph_sigma = tree.pop('posthoc_sigma_rel', None)
    if distill is not None:
        distill = {k: (float(v) if k == 'w' else int(v)) for k, v in distill.items()}
    if np.ndim(tree['step']) == 1:
        tree = strip_device_axis(tree, 0)
    opt = tree['opt_state']
    if 'count' not in opt['0']:          # chain(clip_by_global_norm, adam(..)): the clip state is empty
        opt = opt['1']
    adam, sched = opt['0'], opt['1']
    if 'count' in sched and int(sched['count']) != int(adam['count']):
        raise ValueError(f"schedule count {int(sched['count'])} differs from the Adam count {int(adam['count'])}")
    out = {'step': int(tree['step']), 'count': int(adam['count']), 'skipped': 0 if skipped is None else int(skipped),
           'prediction': prediction, 'distill': distill}
    for k, sub in (('params', tree['params']), ('mu', adam['mu']), ('nu', adam['nu']), ('ema', tree.get('ema_params'))):
        out[k] = None if sub is None else pack_flat(sub, spec, nparams)
    ph = tree.get('posthoc_ema')
    out['posthoc'] = None if ph is None else tuple(pack_flat(ph[k], spec, nparams) for k in ('0', '1'))
    out['posthoc_sigma_rel'] = None if ph_sigma is None else tuple(float(x) for x in np.asarray(ph_sigma).reshape(-1))
    out['rng'] = None if rng is None else [rng[str(r)] for r in range(len(rng))]
    return out


def save_train_state(ckpt_dir: str, state, step: int, prefix: str = 'state', overwrite: bool = True,
                     add_device_axis: bool = False) -> str:
    """Writes the whole TrainState -- params, Adam mu / nu / count, step, ema_params when the state keeps an EMA, the two
    post-hoc averages and their sigma_rel when it keeps them, the count
    of skipped updates when it clips or warms up, the state's prediction ('eps' or 'v'), a distilled student's record
    (state.distill) and the host cond_mask stream of
    every rank -- to f'{prefix}{step}' in ckpt_dir (layout: train_state_tree).  The file stays a
    valid params checkpoint: restore_checkpoint(ckpt_dir, prefix=prefix) returns its params tree.

    Under torch.distributed this is collective: every rank must call it; the cond_mask streams are gathered and rank 0
    writes.  The tree is built in host memory before it is written (about 7 GB for the full 439 M-parameter model with an
    EMA, 8.8 GB with the post-hoc averages).  Returns the file path."""
    from . import dist as xdist
    rngs = xdist.all_gather_object(rng_state_dict(state._mask_rng, state._frozen_mask))
    path = os.path.join(ckpt_dir, f'{prefix}{step}')
    if xdist.rank() == 0:
        spec = state.params.spec

        def host(t):
            return leaf_tree(t.detach().cpu().numpy(), spec)
        tree = train_state_tree(host(state.params.flat), host(state.opt_state.mu), host(state.opt_state.nu),
                                state.opt_state.count, state.step,
                                ema=None if state.ema_params is None else host(state.ema_params.flat),
                                rng=rngs, add_device_axis=add_device_axis, clip=state.tx.max_grad_norm is not None,
                                schedule=state.tx.warmup_steps > 0,
                                skipped=state.skipped_steps if state.clip is not None else None,
                                prediction=state.prediction, distill=state.distill,
                                posthoc=None if state.posthoc is None else tuple(host(f) for f in state.posthoc.flats()),
                                posthoc_sigma_rel=None if state.posthoc is None else state.posthoc.sigma_rel)
        path = save_checkpoint(ckpt_dir, tree, step, prefix=prefix, overwrite=overwrite)
    xdist.barrier()
    return path


def restore_train_state(ckpt_dir: str, state, prefix: str = 'state'):
    """Restores the latest f'{prefix}<step>' file (or the file `ckpt_dir`) written by save_train_state INTO `state`, a
    TrainState from create_train_state with the same model, batch size and image side, and returns it (None if there is
    no such file).

    The flat device buffers are overwritten in place, never rebound, so a TrainStep already built (and CUDA-graph-captured)
    on `state` stays valid; it re-derives its device step counter and dropout seed from the restored count.  A file without
    EMA restored into a state with one starts the EMA from the restored params; a file with an EMA restored into a state
    without one ignores it.  The clipping / warm-up settings are those of `state`, whatever the file was written with; the
    skip counter is restored (0 if the file has none).  A file whose prediction ('eps' when it records none) differs from
    the state's raises ValueError before anything is written: a v model resumed as an eps one (or the reverse) would be
    trained on the other target.  Likewise a file whose distillation record (None when it has none) differs from the state's:
    a student resumed for another teacher grid, round or guidance would be trained on other targets.  A state with post-hoc
    averages takes them from the file, which must hold averages of the same sigma_rel (ValueError otherwise, before anything
    is written: averages started mid-run would not follow the power profiles reconstruction assumes); a file with averages
    restored into a state without them ignores them.  Each rank takes its own cond_mask stream; if the world size differs from the saved one the
    freshly seeded streams are kept (with a warning), and a resume is then no longer bit-exact."""
    from . import dist as xdist
    path = ckpt_dir if os.path.isfile(ckpt_dir) else latest_checkpoint(ckpt_dir, prefix)
    if path is None:
        return None
    with open(path, 'rb') as fh:
        tree = msgpack_restore(fh.read())
    r = parse_train_state_tree(tree, state.params.spec, state.params.flat.numel())
    if r['prediction'] != state.prediction:
        raise ValueError(f"{path}: the checkpoint holds a prediction={r['prediction']!r} model, the state trains "
                         f"prediction={state.prediction!r}")
    if r['distill'] != state.distill:
        raise ValueError(f"{path}: the checkpoint holds a model with distillation record {r['distill']}, the state trains "
                         f"one with {state.distill}")
    if state.posthoc is not None and r['posthoc_sigma_rel'] != tuple(state.posthoc.sigma_rel):
        held = 'no post-hoc averages' if r['posthoc'] is None else f"post-hoc averages of sigma_rel {r['posthoc_sigma_rel']}"
        raise ValueError(f'{path}: the checkpoint holds {held}, the state keeps sigma_rel {state.posthoc.sigma_rel}')
    state.params.flat.copy_(r['params'])
    state.opt_state.mu.copy_(r['mu'])
    state.opt_state.nu.copy_(r['nu'])
    if state.ema_params is not None:
        state.ema_params.flat.copy_(r['ema'] if r['ema'] is not None else r['params'])
    if state.posthoc is not None:
        for f, saved in zip(state.posthoc.flats(), r['posthoc']):
            f.copy_(saved)
    if state.clip is not None:
        state.clip.skipped.fill_(r['skipped'])
    state.step = r['step']
    state.opt_state.count = r['count']
    world = xdist.world_size()
    if r['rng'] is None or len(r['rng']) != world:
        saved = 'no' if r['rng'] is None else len(r['rng'])
        warnings.warn(f'{path}: cond_mask streams saved for {saved} ranks, running on {world}: keeping the fresh streams '
                      f'(the resumed run is not bit-identical to an uninterrupted one)')
    else:
        state._frozen_mask = _set_rng_state(state._mask_rng, r['rng'][xdist.rank()])
    return state
