"""fp64 restatement of the post-hoc EMA (Karras et al. 2024, §3), written from the definitions and independent of
novel_view_synthesis_3d_b200.posthoc: the power-average recursion, the weights it gives each update, the closed-form
profile inner products, the Gram matrix and the least-squares solve, and the float32 update the Adam kernel applies."""
import numpy as np


def sigma_rel(gamma: float) -> float:
    return np.sqrt(gamma + 1.0) / ((gamma + 2.0) * np.sqrt(gamma + 3.0))


def gamma_of(sr: float) -> float:
    """gamma > 0 with sigma_rel(gamma) = sr, by bisection (sigma_rel decreases on gamma > 0)."""
    lo, hi = 0.0, 1e6
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if sigma_rel(mid) > sr else (lo, mid)
    return 0.5 * (lo + hi)


def beta(t: int, gamma: float) -> float:
    return (1.0 - 1.0 / t) ** (gamma + 1.0)


def recursion_weights(T: int, gamma: float) -> np.ndarray:
    """Weight of theta_0 (the initial weights) .. theta_T in the average after T updates, by running the recursion."""
    w = np.zeros(T + 1)
    w[0] = 1.0
    for t in range(1, T + 1):
        b = beta(t, gamma)
        w *= b
        w[t] += 1.0 - b
    return w


def closed_form_weights(T: int, gamma: float) -> np.ndarray:
    tau = np.arange(1, T + 1, dtype=np.float64)
    return np.concatenate([[0.0], (tau ** (gamma + 1) - (tau - 1) ** (gamma + 1)) / float(T) ** (gamma + 1)])


def inner(ti, gi, tj, gj) -> float:
    """<p_i, p_j> = integral over (0, min(t_i, t_j)] of (g_i+1) x^g_i / t_i^(g_i+1) * (g_j+1) x^g_j / t_j^(g_j+1) dx."""
    m = min(ti, tj)
    return (gi + 1) * (gj + 1) * m ** (gi + gj + 1) / ((gi + gj + 1) * float(ti) ** (gi + 1) * float(tj) ** (gj + 1))


def coefficients(in_t, in_g, t, g) -> np.ndarray:
    A = np.array([[inner(a, ga, b, gb) for b, gb in zip(in_t, in_g)] for a, ga in zip(in_t, in_g)])
    b = np.array([inner(a, ga, t, g) for a, ga in zip(in_t, in_g)])
    return np.linalg.lstsq(A, b, rcond=None)[0]


def trajectory(T: int, d: int = 64, seed: int = 0) -> np.ndarray:
    """theta_1 .. theta_T of the synthetic experiment: sin(tau f / 3000) + 0.3 noise, one frequency f per coordinate."""
    rng = np.random.default_rng(seed)
    f = rng.uniform(0.5, 3.0, d)
    tau = np.arange(1, T + 1, dtype=np.float64)[:, None]
    return np.sin(tau * f / 3000.0) + 0.3 * rng.standard_normal((T, d))


def run_averages(theta: np.ndarray, gammas, every: int):
    """Runs the recursion of every gamma over theta (initial weights: zeros, which beta_1 = 0 discards) and returns the
    snapshots [(t, gamma, average)] taken every `every` updates."""
    e = [np.zeros(theta.shape[1]) for _ in gammas]
    out = []
    for t in range(1, theta.shape[0] + 1):
        for k, g in enumerate(gammas):
            b = beta(t, g)
            e[k] = b * e[k] + (1.0 - b) * theta[t - 1]
        if t % every == 0:
            out += [(t, g, e[k].copy()) for k, g in enumerate(gammas)]
    return out


def exact_average(theta: np.ndarray, t: int, gamma: float) -> np.ndarray:
    return closed_form_weights(t, gamma)[1:] @ theta[:t]


def f32_update(e: np.ndarray, p_new: np.ndarray, t: int, gamma: float) -> np.ndarray:
    """The kernel's float32 update: beta and 1 - beta formed in double and rounded once, each product and the sum rounded."""
    b = beta(t, gamma)
    bf, omb = np.float32(b), np.float32(1.0 - b)
    return (bf * e.astype(np.float32) + omb * p_new.astype(np.float32)).astype(np.float32)
