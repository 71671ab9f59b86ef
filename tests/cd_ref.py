"""float64 restatement of consistency distillation (novel_view_synthesis_3d_b200.distill.ConsistencyTeacher, csrc/cd.cu): the
teacher's DDIM chain f(z, n) from grid position n to clean, one training target (teacher step, target network, target
formula), and multistep consistency sampling, all on explicit sampler-table rows and an explicit denoiser."""
import math

import numpy as np

from tests import solver_ref as SR

C_RECIP, C_RECIPM1, C_X0, C_Z, SIGMA, LOGSNR, C_PREV = range(7)


def exact_out(z, ac, prediction, mu=SR.MU, s=SR.SD):
    """The exact eps (or v) of per-pixel Gaussian data N(mu, s^2) at alpha-bar ac."""
    eps = SR.exact_eps(z, ac, mu=mu, s=s)
    if prediction == 'eps':
        return eps
    x0 = (z - math.sqrt(1. - ac) * eps) / math.sqrt(ac)
    return math.sqrt(ac) * eps - math.sqrt(1. - ac) * x0


def teacher_fn(prediction, w):
    """teacher(z, t): the (guided) output of the exact conditional denoiser at timestep t; guided against a different
    "unconditional" Gaussian when w is a float."""
    ac_full = SR.alphas_cumprod()

    def teacher(z, t):
        a = ac_full[t]
        oc = exact_out(z, a, prediction)
        if w is None:
            return oc
        return (1 + w) * oc - w * exact_out(z, a, prediction, mu=-0.05, s=0.25)
    return teacher


def table_step(row, out, z, noise=0.0):
    """The fixed-clip table step in fp64: x0 = clip(c_recip z - c_recipm1 out), z' = c_x0 x0 + c_z z + sigma noise.
    Returns (z', x0)."""
    x0 = np.clip(row[C_RECIP] * z - row[C_RECIPM1] * out, -1., 1.)
    return row[C_X0] * x0 + row[C_Z] * z + row[SIGMA] * noise, x0


def ddim_chain(z, n, grid, ttab, teacher):
    """f(z, n): the teacher's DDIM chain on its table from grid position n to clean (the last row lands on x0)."""
    for k in range(n, len(grid)):
        z, _ = table_step(ttab[k], teacher(z, grid[k]), z)
    return z


def student_v(z, n, grid, ttab, teacher):
    """The v output of a perfect consistency student at position n: alpha_n z - sigma_n v = f(z, n)."""
    a = SR.alphas_cumprod()[grid[n]]
    return (math.sqrt(a) * z - ddim_chain(z, n, grid, ttab, teacher)) / math.sqrt(1. - a)


def position_of_logsnr(grid, logsnr):
    """The grid position whose timestep has this log-SNR (the target network knows t only through its log-SNR input)."""
    from novel_view_synthesis_3d_b200.sampling import logsnr_schedule_cosine
    ls = logsnr_schedule_cosine(np.asarray(grid) / 1000.0)
    k = int(np.argmin(np.abs(ls - logsnr)))
    assert ls[k] == logsnr, (logsnr, ls[k])
    return k


def cd_target(z, n, grid, ttab, gtab, teacher, target_net):
    """One consistency-distillation target, as xunet_cd_teacher_step, the target forward and xunet_cd_target compute it:
    z^ = row n of the teacher table applied to the teacher's output at (z, t_n); v- = target_net(z^, log-SNR from row n,
    column 5); x0- = clip(a z^ - b v-); v* = (alpha_n z - x0-) / sigma_n.  Returns (v*, z^, the target log-SNR)."""
    z_hat, _ = table_step(ttab[n], teacher(z, grid[n]), z)
    logsnr = ttab[n, LOGSNR]
    v_minus = target_net(z_hat, logsnr)
    a, b, alpha, sigma = gtab[n]
    x0 = np.clip(a * z_hat - b * v_minus, -1., 1.)
    return (alpha * z - x0) / sigma, z_hat, logsnr


def consistency_sample(z, grid_k, rows, student, noises):
    """Multistep consistency sampling on the table rows of consistency_grid timesteps grid_k (loop order): per step the
    student's output at (z, t_k), then the table step with noise noises[k]."""
    for k in range(len(grid_k)):
        z, _ = table_step(rows[k], student(z, k), z, noises[k])
    return z
