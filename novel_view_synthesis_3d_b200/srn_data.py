"""SRN (cars / chairs) scene reader for the X-UNet training / sampling loops  (SURVEY 8(f) row 3).

Produces exactly the batch contract of the reference's `SceneClassDataset` (dataset/data_loader.py:102-113, collate :163-181):
    x      (B,S,S,3) float32 in [-1,1]   source view                        R1,t1  its cam->world pose
    target (B,S,S,3) float32 in [-1,1]   a random second view of the scene  R2,t2  its cam->world pose
    K      (B,3,3)   pixel intrinsics rescaled to S
and, with `host_diffusion=True`, also z / noise / logsnr computed on the host like the reference (float64); otherwise those
are left to `ForwardDiffusion` on the GPU.  Decoding uses OpenCV only (the reference needs imageio + skimage, absent here):
`load_rgb` = first 3 channels -> float32/255 -> centre square crop -> cv2.INTER_AREA resize -> *2-1  (data_util.py:12-24,67-72),
`load_pose` = 4x4 text matrix in one or four lines (data_util.py:43-52), `parse_intrinsics` (util.py:46-81).
Directory layout: <root>/<instance>/{rgb/*.png, pose/*.txt, intrinsics.txt}.
"""
from __future__ import annotations

import os
import queue
import threading
from glob import glob
from typing import Dict, Iterator, List, Optional

import numpy as np

from .sampling import cosine_beta_schedule, logsnr_schedule_cosine

_IMG_EXT = ('*.png', '*.jpg', '*.JPEG', '*.JPG')


def load_rgb(path: str, sidelength: Optional[int] = None) -> np.ndarray:
    """-> (S,S,3) float32 in [-1,1], RGB order, HWC (the reference returns CHW and transposes back, data_loader.py:102)."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(path)
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, axis=2)
    img = img[:, :, :3][:, :, ::-1]                                   # BGR(A) -> RGB
    scale = 65535.0 if img.dtype == np.uint16 else 255.0
    img = img.astype(np.float32) / scale
    h, w = img.shape[:2]
    m = min(h, w)
    cy, cx = h // 2, w // 2
    img = img[cy - m // 2: cy + m // 2, cx - m // 2: cx + m // 2]      # centre square crop (data_util.py:67-72)
    if sidelength is not None and img.shape[0] != sidelength:
        img = cv2.resize(np.ascontiguousarray(img), (sidelength, sidelength), interpolation=cv2.INTER_AREA)
    return np.ascontiguousarray((img - 0.5) * 2.0, dtype=np.float32)


def load_pose(path: str) -> np.ndarray:
    """4x4 cam->world matrix stored as 16 numbers on one line or as four lines of four."""
    vals = np.array(open(path).read().split(), dtype=np.float32)
    if vals.size < 16:
        raise ValueError(f'{path}: expected 16 numbers, found {vals.size}')
    return vals[:16].reshape(4, 4)


def parse_intrinsics(path: str, trgt_sidelength: Optional[int] = None) -> np.ndarray:
    """intrinsics.txt: line 1 `f cx cy _`, line 4 `height width`  ->  3x3 K rescaled to trgt_sidelength (util.py:46-81)."""
    with open(path) as fh:
        f, cx, cy, _ = map(float, fh.readline().split())
        fh.readline()                      # grid barycenter (unused on this path)
        fh.readline()                      # scale
        height, width = map(float, fh.readline().split())
    if trgt_sidelength is not None:
        cx = cx / width * trgt_sidelength
        cy = cy / height * trgt_sidelength
        f = trgt_sidelength / height * f
    return np.array([[f, 0., cx], [0., f, cy], [0., 0., 1.]], dtype=np.float32)


class SRNScenes:
    """All (instance, view) pairs under root_dir.  Item i = view i as source + a uniformly random view of the same instance
    as target (data_loader.py:88-90)."""

    def __init__(self, root_dir: str, img_sidelength: int = 64, max_num_instances: int = -1,
                 max_observations_per_instance: int = -1, host_diffusion: bool = False, seed: int = 0):
        self.S = img_sidelength
        self.host_diffusion = host_diffusion
        self.rng = np.random.RandomState(seed)
        dirs = sorted(d for d in glob(os.path.join(root_dir, '*/')) if os.path.isdir(os.path.join(d, 'rgb')))
        if not dirs:
            raise AssertionError('No objects in the data directory')        # data_loader.py:130
        if max_num_instances != -1:
            dirs = dirs[:max_num_instances]
        self.instances: List[Dict] = []
        self.index: List[tuple] = []
        for d in dirs:
            imgs = sorted(sum((glob(os.path.join(d, 'rgb', e)) for e in _IMG_EXT), []))
            poses = sorted(glob(os.path.join(d, 'pose', '*.txt')))
            if max_observations_per_instance != -1 and len(imgs) > max_observations_per_instance:
                pick = np.linspace(0, len(imgs), num=max_observations_per_instance, endpoint=False, dtype=int)   # :62-65
                imgs, poses = [imgs[i] for i in pick], [poses[i] for i in pick]
            if len(imgs) != len(poses) or not imgs:
                raise ValueError(f'{d}: {len(imgs)} images vs {len(poses)} poses')
            K = parse_intrinsics(os.path.join(d, 'intrinsics.txt'), self.S)
            self.instances.append(dict(name=os.path.basename(os.path.normpath(d)), imgs=imgs, poses=poses, K=K))
            self.index += [(len(self.instances) - 1, v) for v in range(len(imgs))]
        if host_diffusion:
            ac = np.cumprod(1. - cosine_beta_schedule(1000), axis=0)
            self.sqrt_ac, self.sqrt_1mac = np.sqrt(ac), np.sqrt(1. - ac)

    def __len__(self) -> int:
        return len(self.index)

    def __getitem__(self, i: int) -> Dict[str, np.ndarray]:
        inst_id, v = self.index[i]
        inst = self.instances[inst_id]
        v2 = int(self.rng.randint(len(inst['imgs'])))
        p1, p2 = load_pose(inst['poses'][v]), load_pose(inst['poses'][v2])
        item = dict(x=load_rgb(inst['imgs'][v], self.S), target=load_rgb(inst['imgs'][v2], self.S),
                    R1=p1[:3, :3].copy(), t1=p1[:3, 3].copy(), R2=p2[:3, :3].copy(), t2=p2[:3, 3].copy(), K=inst['K'])
        if self.host_diffusion:            # data_loader.py:90-110 (float64 like the reference)
            noise = self.rng.randn(self.S, self.S, 3)
            t = int(self.rng.randint(0, 1000))
            item['z'] = self.sqrt_ac[t] * item['target'] + self.sqrt_1mac[t] * noise
            item['noise'] = noise
            item['logsnr'] = float(logsnr_schedule_cosine(t / 1000.0))
        return item

    def instance_views(self, i: int) -> Dict:
        """Every view of instance i, in the reader's sorted file order (index j = the j-th file kept after
        max_observations_per_instance): dict(name, x (n,S,S,3), R (n,3,3), t (n,3), K (3,3)).  Draws nothing from self.rng,
        so it leaves the training stream of batches() unchanged (evaluation reads held-out views this way)."""
        inst = self.instances[i]
        poses = np.stack([load_pose(p) for p in inst['poses']])
        return dict(name=inst['name'], x=np.stack([load_rgb(p, self.S) for p in inst['imgs']]),
                    R=np.ascontiguousarray(poses[:, :3, :3]), t=np.ascontiguousarray(poses[:, :3, 3]), K=inst['K'])

    @staticmethod
    def collate(items: List[Dict[str, np.ndarray]]) -> Dict[str, np.ndarray]:
        return {k: np.stack([np.asarray(it[k]) for it in items]) for k in items[0]}

    def batches(self, batch_size: int, shuffle: bool = True, drop_last: bool = True, prefetch: int = 2) -> Iterator[Dict]:
        """Endless stream of collated batches (train.py's `cycle(DataLoader(...))`), decoded by a background thread."""
        q: "queue.Queue" = queue.Queue(maxsize=prefetch)

        def work():
            while True:
                order = self.rng.permutation(len(self)) if shuffle else np.arange(len(self))
                for s in range(0, len(order), batch_size):
                    idx = order[s:s + batch_size]
                    if len(idx) < batch_size and drop_last:
                        continue
                    q.put(self.collate([self[int(j)] for j in idx]))

        threading.Thread(target=work, daemon=True).start()
        while True:
            yield q.get()


# ---- device-resident training data --------------------------------------------------------------------------------------
# DeviceScenes holds every view of an SRN tree in GPU memory; xunet_srn_batch (csrc/data.cu) draws, gathers and noises one
# micro-batch from it inside the training step.  The draw order is a function of (seed, Adam count, micro-batch, rank), so a
# resumed run sees the same data as an uninterrupted one.  The functions below restate the kernel's draw in numpy.

_M64 = 0xFFFFFFFFFFFFFFFF


def _u64(x) -> np.ndarray:
    return np.asarray(x, dtype=np.uint64) if not isinstance(x, int) else np.asarray(x & _M64, dtype=np.uint64)


def mix64(z) -> np.ndarray:
    """xu_mix64 (csrc/common.cuh) on uint64 arrays, wrapping like the device."""
    z = _u64(z)
    with np.errstate(over='ignore'):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _add(a, b) -> np.ndarray:
    with np.errstate(over='ignore'):
        return _u64(a) + _u64(b)


def permute(x, n: int, seed: int, epoch) -> np.ndarray:
    """P_{seed,epoch}(x) of the kernel (srn_permute): a keyed 4-round Feistel bijection of [0, 4^h) with 4^h >= n, h >= 1,
    cycle-walked back into [0, n).  x, epoch: integer arrays (broadcast together)."""
    x, epoch = np.broadcast_arrays(_u64(x), _u64(epoch))
    h = 1
    while (1 << (2 * h)) < n:
        h += 1
    mask, hh = np.uint64((1 << h) - 1), np.uint64(h)
    with np.errstate(over='ignore'):
        base = mix64(_u64(seed) ^ np.uint64(0x243F6A8885A308D3))
        keys = [mix64(base + epoch * np.uint64(4) + np.uint64(r)) for r in range(4)]

    def rounds(y, ks):
        L, R = y >> hh, y & mask
        for k in ks:
            L, R = R, L ^ (mix64(R ^ k) & mask)
        return (L << hh) | R

    y = rounds(x.copy(), keys)
    out = y >= np.uint64(n)
    while out.any():
        y[out] = rounds(y[out], [k[out] for k in keys])
        out = y >= np.uint64(n)
    return y


def diffusion_seed(seed: int, count: int, j: int, k: int, rank: int) -> int:
    """Forward-diffusion seed of micro-batch j of the update at Adam count `count` on `rank` (srn_diffusion_seed)."""
    mb = (int(count) * int(k) + int(j)) & _M64
    s = mix64(_add(mix64(_add(mix64(_u64(seed) ^ np.uint64(0xA4093822299F31D0)), mb)), int(rank)))
    return int(s)


def draw_indices(first: np.ndarray, count: np.ndarray, item_inst: np.ndarray, seed: int, c: int, j: int, k: int, rank: int,
                 world: int, B: int) -> np.ndarray:
    """(B, 3) int64 (inst, v, v2) of micro-batch j of the update at Adam count c on `rank` of `world`: draw index
    g = ((c k + j) world + rank) B + b, source item P_{seed, g // N}(g mod N), target view mix(seed, g) mod count[inst]."""
    n = len(item_inst)
    base = ((int(c) * k + j) * world + rank) * B
    g = np.array([(base + b) & _M64 for b in range(B)], dtype=np.uint64)
    item = permute(g % np.uint64(n), n, seed, g // np.uint64(n)).astype(np.int64)
    inst = item_inst[item].astype(np.int64)
    h = mix64(_add(mix64(_u64(seed) ^ np.uint64(0x13198A2E03707344)), g))
    v2 = (h % count[inst].astype(np.uint64)).astype(np.int64)
    return np.stack([inst, item - first[inst], v2], axis=1)


def load_rgb_u8(path: str, sidelength: int) -> Optional[np.ndarray]:
    """load_rgb's 8-bit RGB centre crop (S,S,3) uint8 when the file is an 8-bit PNG whose crop is already S x S (so load_rgb
    would not resize it); None otherwise.  u8_to_float(load_rgb_u8(p, S)) equals load_rgb(p, S) bit for bit."""
    import cv2
    if not path.lower().endswith('.png'):
        return None
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(path)
    if img.dtype != np.uint8:
        return None
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, axis=2)
    img = img[:, :, :3][:, :, ::-1]
    h, w = img.shape[:2]
    m = min(h, w)
    cy, cx = h // 2, w // 2
    img = img[cy - m // 2: cy + m // 2, cx - m // 2: cx + m // 2]
    if img.shape[:2] != (sidelength, sidelength):
        return None
    return np.ascontiguousarray(img)


def u8_to_float(u: np.ndarray) -> np.ndarray:
    """((u / 255) - 0.5) * 2 in float32, one rounding per operation: load_rgb's arithmetic, and the kernel's."""
    return (u.astype(np.float32) / np.float32(255.0) - np.float32(0.5)) * np.float32(2.0)


def scene_files(ds: SRNScenes) -> List[str]:
    """Every file a decode of `ds` reads, in order (views, poses, intrinsics per instance)."""
    out = []
    for inst in ds.instances:
        out += [os.path.abspath(p) for p in inst['imgs']] + [os.path.abspath(p) for p in inst['poses']]
        out.append(os.path.abspath(os.path.join(os.path.dirname(os.path.dirname(inst['imgs'][0])), 'intrinsics.txt')))
    return out


def decode_scenes(ds: SRNScenes, workers: int = 8) -> Dict[str, np.ndarray]:
    """Decodes every view of `ds` once, on a thread pool (cv2 releases the GIL).  Host only.  Returns
    pixels (N,S,S,3) uint8 when every view is an 8-bit PNG whose centre crop is S x S, else float32 (load_rgb's output);
    R (N,3,3), t (N,3) float32; K (I,3,3) float32; first, count (I,) int32; item_inst (N,) int32; storage 'uint8' / 'float32'."""
    from concurrent.futures import ThreadPoolExecutor
    S = ds.S
    imgs = [p for inst in ds.instances for p in inst['imgs']]
    poses = [p for inst in ds.instances for p in inst['poses']]

    def one(path):
        u = load_rgb_u8(path, S)
        return u if u is not None else load_rgb(path, S)

    with ThreadPoolExecutor(max_workers=max(1, int(workers))) as ex:
        views = list(ex.map(one, imgs))
        pose = np.stack(list(ex.map(load_pose, poses)))
    if all(v.dtype == np.uint8 for v in views):
        pixels, storage = np.stack(views), 'uint8'
    else:
        pixels = np.stack([u8_to_float(v) if v.dtype == np.uint8 else v for v in views]).astype(np.float32, copy=False)
        storage = 'float32'
    counts = np.array([len(inst['imgs']) for inst in ds.instances], dtype=np.int32)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)
    return dict(pixels=pixels, storage=storage, R=np.ascontiguousarray(pose[:, :3, :3], dtype=np.float32),
                t=np.ascontiguousarray(pose[:, :3, 3], dtype=np.float32),
                K=np.stack([inst['K'] for inst in ds.instances]).astype(np.float32), first=first, count=counts,
                item_inst=np.repeat(np.arange(len(counts), dtype=np.int32), counts))


_CACHE_ARRAYS = ('pixels', 'R', 't', 'K', 'first', 'count', 'item_inst')
_CACHE_VERSION = 1


def load_or_decode(ds: SRNScenes, cache: Optional[str] = None, workers: int = 8,
                   max_observations_per_instance: int = -1):
    """decode_scenes(ds), read from / written to the cache directory `cache` when given: one .npy per array plus meta.json
    (file list, S, storage kind, max_observations_per_instance).  A cache whose meta.json does not match is decoded again and
    overwritten.  Files are written under temporary names and renamed, meta.json last.  Returns (arrays, read_from_cache)."""
    import json
    meta = dict(version=_CACHE_VERSION, files=scene_files(ds), S=int(ds.S),
                max_observations_per_instance=int(max_observations_per_instance))
    if cache is not None:
        mpath = os.path.join(cache, 'meta.json')
        try:
            with open(mpath) as fh:
                saved = json.load(fh)
            if {k: saved.get(k) for k in meta} == meta:
                arrays = {k: np.load(os.path.join(cache, k + '.npy')) for k in _CACHE_ARRAYS}
                arrays['storage'] = saved['storage']
                if str(arrays['pixels'].dtype) == saved['storage']:
                    return arrays, True
        except (OSError, ValueError, KeyError):
            pass
    arrays = decode_scenes(ds, workers)
    if cache is not None:
        os.makedirs(cache, exist_ok=True)
        tag = f'.tmp{os.getpid()}'
        for k in _CACHE_ARRAYS:
            with open(os.path.join(cache, k + '.npy' + tag), 'wb') as fh:
                np.save(fh, arrays[k])
            os.replace(os.path.join(cache, k + '.npy' + tag), os.path.join(cache, k + '.npy'))
        with open(os.path.join(cache, 'meta.json' + tag), 'w') as fh:
            json.dump(dict(meta, storage=arrays['storage']), fh)
        os.replace(os.path.join(cache, 'meta.json' + tag), os.path.join(cache, 'meta.json'))
    return arrays, False


class DeviceScenes:
    """Every view of an SRN tree decoded once and held in GPU memory, for TrainStep(data=..): each micro-batch is then drawn,
    gathered and forward-diffused by one kernel inside the step (xunet_srn_batch), with no host work and no PCIe traffic.

        store = DeviceScenes('cars_train', 64, max_observations_per_instance=50, cache='cars64.cache')
        step = TrainStep(state, data=store, data_seed=0)
        loss = step()

    root_or_scenes: a directory (read with SRNScenes) or an SRNScenes (its instances and file order are used as they are).
    Pixels are stored as uint8 (N,S,S,3) when every view is an 8-bit PNG whose centre crop is already S x S -- the kernel then
    forms load_rgb's float32 values bit for bit -- and as load_rgb's float32 output otherwise (resized, 16-bit or JPEG views).
    cache: a directory for the decoded arrays (see load_or_decode), so data-parallel ranks and later runs skip the decode.
    The store is checked against torch.cuda.mem_get_info before anything is allocated: a store that does not fit raises
    MemoryError with its size instead of failing halfway."""

    def __init__(self, root_or_scenes, img_sidelength: int, max_observations_per_instance: int = -1, device=None,
                 workers: int = 8, cache: Optional[str] = None):
        import torch
        from . import _lib
        if isinstance(root_or_scenes, SRNScenes):
            ds = root_or_scenes
            if ds.S != img_sidelength:
                raise ValueError(f'the SRNScenes reads views at S = {ds.S}, the store was asked for S = {img_sidelength}')
        else:
            ds = SRNScenes(root_or_scenes, img_sidelength=img_sidelength,
                           max_observations_per_instance=max_observations_per_instance)
        self.S = int(img_sidelength)
        self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device(f'cuda:{torch.cuda.current_device()}')
        arrays, self.from_cache = load_or_decode(ds, cache, workers, max_observations_per_instance)
        self.storage = arrays['storage']
        self.nbytes = sum(int(arrays[k].nbytes) for k in _CACHE_ARRAYS)
        free, total = torch.cuda.mem_get_info(self.device)
        if self.nbytes > free:
            raise MemoryError(f'DeviceScenes needs {self.nbytes} bytes of device memory for {len(arrays["item_inst"])} views at '
                              f'S = {self.S} ({self.storage}); {self.device} has {free} of {total} bytes free')
        self.first, self.count, self.item_inst = arrays['first'], arrays['count'], arrays['item_inst']
        self.n_items, self.n_instances = len(self.item_inst), len(self.first)
        self.names = [inst['name'] for inst in ds.instances]
        dev = {k: torch.from_numpy(np.ascontiguousarray(arrays[k])).to(self.device) for k in _CACHE_ARRAYS}
        self.pixels, self.R, self.t, self.K = dev['pixels'], dev['R'], dev['t'], dev['K']
        self._first, self._count, self._item_inst = dev['first'], dev['count'], dev['item_inst']
        self.c_store = _lib.XunetSrnStore(
            pixels=self.pixels.data_ptr(), pixel_kind=_lib.PIXELS_U8 if self.storage == 'uint8' else _lib.PIXELS_F32,
            S=self.S, n_items=self.n_items, n_instances=self.n_instances, R=self.R.data_ptr(), t=self.t.data_ptr(),
            K=self.K.data_ptr(), first=self._first.data_ptr(), count=self._count.data_ptr(),
            item_inst=self._item_inst.data_ptr())

    def __len__(self) -> int:
        return self.n_items

    def draws(self, count: int, j: int, k: int, rank: int, world: int, B: int, seed: int = 0) -> np.ndarray:
        """(B, 3) (inst, v, v2) that micro-batch j of the update at Adam count `count` draws on `rank` of `world` with
        data_seed `seed` (the host restatement of the kernel's draw)."""
        return draw_indices(self.first, self.count, self.item_inst, seed, count, j, k, rank, world, B)
