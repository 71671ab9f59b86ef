"""In-tree build of libxunet_b200.so for the H100 (sm_90a only; nvcc cross-compiles without a GPU).

The .so and the objects are build products (git-ignored); build() recompiles them whenever the sources or flags change."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / 'csrc'
INCLUDE = ROOT / 'include'
OBJ_DIR = ROOT / 'build' / 'obj'
LIB = PKG / 'libxunet_b200.so'
SOURCES = ['engine.cu', 'kernels_conv.cu', 'kernels_elem.cu', 'kernels_attn.cu', 'conv_tc.cu', 'attn_tc.cu', 'wgrad_tc.cu', 'metrics.cu',
           'sampler.cu', 'data.cu', 'pose_grad.cu', 'distill.cu', 'field.cu', 'pose_fit.cu',
           'lift.cu', 'cd.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = [*ARCH, '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-I', str(INCLUDE), '-I', str(CSRC)]


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    deps = list(CSRC.glob('*.cu')) + list(CSRC.glob('*.cuh')) + list(CSRC.glob('*.h')) + list(INCLUDE.glob('*.h'))
    stamp = OBJ_DIR / 'stamp'
    digest = _digest(deps)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str):
        obj = OBJ_DIR / (src + '.o')
        cmd = [nvcc, *NVCC_FLAGS, '-c', str(CSRC / src), '-o', str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'nvcc failed for {src}:\n{r.stdout}\n{r.stderr}')
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr, file=sys.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, '-shared', '-o', str(LIB), *map(str, objs), *ARCH,
           '-Xcompiler', '-fPIC', '-lcudart_static', '-ldl', '-lrt', '-lpthread']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
    stamp.write_text(digest)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
