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
