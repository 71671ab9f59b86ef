"""Post-hoc EMA (Karras et al. 2024, *Analyzing and Improving the Training Dynamics of Diffusion Models*, §3): choose the EMA
length of the weights after training.

A state built with create_train_state(posthoc_ema=(s_a, s_b)) keeps two power-function averages of the weights, updated in
the fused Adam pass (xunet_adam_posthoc_step).  At Adam count t an average of exponent gamma is

    e_t = beta_t e_{t-1} + (1 - beta_t) theta_t,   beta_t = (1 - 1/t)^(gamma + 1)

so the parameters after update tau carry the weight (tau^(gamma+1) - (tau-1)^(gamma+1)) / t^(gamma+1): exactly the integral
over (tau - 1, tau] of the profile p(tau) = (gamma + 1) tau^gamma / t^(gamma+1), with none left on the initial weights.
save_snapshot writes both averages every so often; reconstruct solves for the least-squares combination of all snapshots'
profiles that best matches the profile of another length (sigma_rel) at any count t up to the last snapshot, and sums the
snapshots with those coefficients.

sigma_rel is the standard deviation of the profile relative to its length t: sigma_rel = (g+1)^(1/2) (g+2)^-1 (g+3)^(-1/2).
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from .checkpoint import leaf_tree, msgpack_restore, msgpack_serialize
from .xunet import ParamTree, _flatten, _nest

SIGMA_REL_MAX = float(1.0 / np.sqrt(12.0))     # sigma_rel at gamma = 0; smaller widths have gamma > 0
SNAPSHOT_PREFIX = 'posthoc'                     # snapshot files: f'{SNAPSHOT_PREFIX}<Adam count>'


def sigma_rel_to_gamma(sigma_rel: float) -> float:
    """Exponent gamma of the power-function profile of relative width sigma_rel in (0, 1/sqrt(12)): the largest real root of
    gamma^3 + 7 gamma^2 + (16 - s^-2) gamma + (12 - s^-2)."""
    s = float(sigma_rel)
    if not (0.0 < s < SIGMA_REL_MAX):
        raise ValueError(f'sigma_rel must lie in (0, {SIGMA_REL_MAX:.4f}), got {sigma_rel}')
    r = np.roots([1.0, 7.0, 16.0 - s ** -2, 12.0 - s ** -2])
    return float(r[np.abs(r.imag) < 1e-9 * (1.0 + np.abs(r.real))].real.max())


def gamma_to_sigma_rel(gamma: float) -> float:
    """Relative width of the power-function profile of exponent gamma > -1."""
    g = float(gamma)
    if not (np.isfinite(g) and g > -1.0):
        raise ValueError(f'gamma must be finite and > -1, got {gamma}')
    return float(np.sqrt(g + 1.0) / ((g + 2.0) * np.sqrt(g + 3.0)))


def check_posthoc_ema(posthoc_ema) -> tuple:
    """create_train_state's posthoc_ema: two different sigma_rel in (0, 1/sqrt(12)).  Returns them as floats."""
    try:
        pair = tuple(float(s) for s in posthoc_ema)
    except TypeError:
        raise ValueError(f'posthoc_ema must be two sigma_rel values, got {posthoc_ema!r}') from None
    if len(pair) != 2:
        raise ValueError(f'posthoc_ema must be two sigma_rel values, got {posthoc_ema!r}')
    for s in pair:
        sigma_rel_to_gamma(s)
    if pair[0] == pair[1]:
        raise ValueError(f'posthoc_ema needs two different sigma_rel values, got {pair}')
    return pair


@dataclass
class PosthocEMA:
    """The two power-function averages a TrainState keeps (create_train_state(posthoc_ema=..)): params-shaped trees over
    their own flat device buffers, with their sigma_rel and gamma."""
    a: ParamTree
    b: ParamTree
    sigma_rel: tuple
    gamma: tuple

    @staticmethod
    def create(model, params: ParamTree, sigma_rel: tuple, S: int, B: int) -> "PosthocEMA":
        """Both averages start as copies of `params` (the first update overwrites them)."""
        a = model.tree_from_flat(params.flat.clone(), S, B)
        b = model.tree_from_flat(params.flat.clone(), S, B)
        return PosthocEMA(a, b, tuple(sigma_rel), tuple(sigma_rel_to_gamma(s) for s in sigma_rel))

    def flats(self) -> List[torch.Tensor]:
        return [self.a.flat, self.b.flat]


# ---- profiles and the least-squares solve (fp64) -----------------------------------------------------------------------
def _log_inner(t_i, g_i, t_j, g_j):
    """log <p_i, p_j> of the profiles (t_i, g_i) and (t_j, g_j), broadcast:
    (g_i+1)(g_j+1) m^(g_i+g_j+1) / ((g_i+g_j+1) t_i^(g_i+1) t_j^(g_j+1)), m = min(t_i, t_j)."""
    m = np.minimum(t_i, t_j)
    return (np.log(g_i + 1.0) + np.log(g_j + 1.0) - np.log(g_i + g_j + 1.0) + (g_i + g_j + 1.0) * np.log(m)
            - (g_i + 1.0) * np.log(t_i) - (g_j + 1.0) * np.log(t_j))


def solve_coefficients(in_t, in_gamma, out_t, out_gamma) -> np.ndarray:
    """Coefficients c (one per input profile) of the least-squares fit sum_i c_i p_i ~ p_out of the profile (out_t,
    out_gamma) by the snapshot profiles (in_t[i], in_gamma[i]): lstsq(A, b) with A_ij = <p_i, p_j> and b_i = <p_i, p_out>,
    in fp64.  out_t / out_gamma may be arrays of one shape: the result then has shape (len(in_t),) + that shape."""
    ti = np.asarray(in_t, np.float64).reshape(-1)
    gi = np.asarray(in_gamma, np.float64).reshape(-1)
    if ti.shape != gi.shape or ti.size == 0:
        raise ValueError(f'in_t and in_gamma must be non-empty and of one length, got {ti.shape} and {gi.shape}')
    to, go = np.broadcast_arrays(np.asarray(out_t, np.float64), np.asarray(out_gamma, np.float64))
    for name, t, g in (('in', ti, gi), ('out', to, go)):
        if not (np.all(np.isfinite(t)) and np.all(t >= 1)):
            raise ValueError(f'{name}_t must be finite counts >= 1, got {t}')
        if not (np.all(np.isfinite(g)) and np.all(g > -1)):
            raise ValueError(f'{name}_gamma must be finite and > -1, got {g}')
    A = np.exp(_log_inner(ti[:, None], gi[:, None], ti[None, :], gi[None, :]))
    b = np.exp(_log_inner(ti[:, None], gi[:, None], to.reshape(1, -1), go.reshape(1, -1)))
    c = np.linalg.lstsq(A, b, rcond=None)[0]
    return c.reshape(ti.shape + to.shape)


# ---- snapshots -----------------------------------------------------------------------------------------------------------
def snapshot_record(count: int, sigma_rel, gamma, a: dict, b: dict) -> dict:
    """The tree one snapshot file holds: the Adam count, both sigma_rel and gamma (fp64) and both averages (params-shaped
    trees of fp32 arrays)."""
    return {'count': np.asarray(count, np.int64), 'sigma_rel': np.asarray(sigma_rel, np.float64),
            'gamma': np.asarray(gamma, np.float64), 'a': a, 'b': b}


def save_snapshot(ckpt_dir: str, state) -> Optional[str]:
    """Writes both averages of `state` (a TrainState built with posthoc_ema) at its current Adam count to
    f'posthoc<count>' in ckpt_dir, in the Flax msgpack format of checkpoint.py.  Earlier snapshots are kept.  Every rank
    holds the same averages, so only rank 0 writes; the other ranks return None.  About 2 x 1.76 GB for the full
    439 M-parameter model."""
    from . import dist as xdist
    ph = state.posthoc
    if ph is None:
        raise ValueError('the state keeps no post-hoc EMA: build it with create_train_state(posthoc_ema=(s_a, s_b))')
    if xdist.rank() != 0:
        return None
    count = int(state.opt_state.count)
    host = lambda t: leaf_tree(t.detach().float().cpu().numpy(), state.params.spec)
    rec = snapshot_record(count, ph.sigma_rel, ph.gamma, host(ph.a.flat), host(ph.b.flat))
    os.makedirs(ckpt_dir, exist_ok=True)
    path = os.path.join(ckpt_dir, f'{SNAPSHOT_PREFIX}{count}')
    tmp = path + '.tmp'
    with open(tmp, 'wb') as fh:
        fh.write(msgpack_serialize(rec))
    os.replace(tmp, path)
    return path


@dataclass
class Snapshot:
    """One snapshot file: its path, Adam count t, sigma_rel and gamma of both averages, and the parameter leaves' shapes."""
    path: str
    t: int
    sigma_rel: tuple
    gamma: tuple
    shapes: dict

    def averages(self):
        """(a, b): both averages as nested dicts of fp32 arrays (reads the file)."""
        rec = _read(self.path)
        return rec['a'], rec['b']


def _read(path: str) -> dict:
    with open(path, 'rb') as fh:
        rec = msgpack_restore(fh.read())
    if not isinstance(rec, dict) or not {'count', 'sigma_rel', 'gamma', 'a', 'b'} <= set(rec):
        raise ValueError(f'{path} is not a post-hoc EMA snapshot')
    return rec


def load_snapshots(ckpt_dir: str) -> List[Snapshot]:
    """Every f'posthoc<count>' snapshot in ckpt_dir, in order of count (each file is read once; the averages are not kept).
    Raises FileNotFoundError when there is none, ValueError when their parameter leaves disagree."""
    found = []
    if os.path.isdir(ckpt_dir):
        for f in os.listdir(ckpt_dir):
            m = re.fullmatch(SNAPSHOT_PREFIX + r'(\d+)', f)
            if m:
                found.append((int(m.group(1)), os.path.join(ckpt_dir, f)))
    if not found:
        raise FileNotFoundError(f'no {SNAPSHOT_PREFIX}<count> snapshot in {ckpt_dir}')
    snaps = []
    for _, path in sorted(found):
        rec = _read(path)
        shapes = {k: tuple(np.shape(v)) for k, v in _flatten(rec['a']).items()}
        if {k: tuple(np.shape(v)) for k, v in _flatten(rec['b']).items()} != shapes:
            raise ValueError(f'{path}: the two averages have different parameter leaves')
        snaps.append(Snapshot(path, int(rec['count']), tuple(float(x) for x in rec['sigma_rel']),
                              tuple(float(x) for x in rec['gamma']), shapes))
    n0 = sum(int(np.prod(s)) for s in snaps[0].shapes.values())
    for s in snaps[1:]:
        if s.shapes != snaps[0].shapes:
            n = sum(int(np.prod(x)) for x in s.shapes.values())
            raise ValueError(f'{s.path} holds {n} parameters in {len(s.shapes)} leaves, {snaps[0].path} holds {n0} in '
                             f'{len(snaps[0].shapes)}: the snapshots are not of one model')
    return snaps


def reconstruct(ckpt_dir: str, sigma_rel: float, t: Optional[int] = None, *, device=None) -> dict:
    """The power-function EMA of relative width sigma_rel at Adam count t (default: the last snapshot's), rebuilt from the
    snapshots in ckpt_dir: c = solve_coefficients over both averages of every snapshot, then sum_i c_i snapshot_i accumulated
    in fp64 on `device` (default cuda) in snapshot order, one snapshot file in host memory at a time, rounded once to fp32.
    Returns a params tree (nested dict of fp32 numpy arrays) that save_checkpoint writes like model<step>.  Raises ValueError
    for a t after the last snapshot."""
    g_out = sigma_rel_to_gamma(sigma_rel)
    snaps = load_snapshots(ckpt_dir)
    t_last = snaps[-1].t
    t = t_last if t is None else int(t)
    if not 1 <= t <= t_last:
        raise ValueError(f't = {t} lies outside [1, {t_last}], the counts the snapshots cover')
    in_t = [s.t for s in snaps for _ in range(2)]
    in_g = [g for s in snaps for g in s.gamma]
    coef = solve_coefficients(in_t, in_g, t, g_out)
    device = torch.device('cuda' if device is None else device)
    names = sorted(snaps[0].shapes)
    acc = None
    for i, s in enumerate(snaps):
        la, lb = (_flatten(x) for x in s.averages())
        if acc is None:
            acc = {k: torch.zeros(snaps[0].shapes[k], dtype=torch.float64, device=device) for k in names}
        for k in names:
            for leaves, c in ((la, coef[2 * i]), (lb, coef[2 * i + 1])):
                acc[k].add_(torch.as_tensor(np.asarray(leaves[k])).to(device).double(), alpha=float(c))
        del la, lb
    return _nest({k: acc[k].float().cpu().numpy() for k in names})
