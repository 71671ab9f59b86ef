"""DDPM ancestral sampler with classifier-free guidance (reference sampling.py:16-53, 73-76, 119-151) on the CUDA path.

Reference behaviour (steps=1000, w=3): per step two model evaluations (cond_mask=1 / 0) -- here ONE forward of a 2B batch
[cond ; uncond] -- eps=(1+w)eps_c-w eps_u, x0=clip(predict_start_from_noise), posterior mean/variance, z<-mean+sigma*N(0,1)
(no noise at t=0), and the log-SNR fed to the network lags one step and starts at -20 (sampling.py:126,151).
`steps<1000` re-spaces the schedule (strided alpha-bar), which is what the 256-step metric uses.

Two samplers that need only tens of steps run through the same device-table step: DDIM (Song et al. 2021; eta = 0
deterministic, eta = 1 the DDPM posterior) and DPM-Solver++(2M) (Lu et al. 2022), a second-order multistep solver in x0
that keeps the previous step's clipped x0 on the device.  Both feed the network the log-SNR of the timestep z is at.
Any of the three can replace the fixed clip of x0 with per-view dynamic thresholding (Imagen, Saharia et al. 2022).

Every sampler reads the network output as eps by default.  prediction='v' reads it as v = sqrt(abar) eps - sqrt(1 - abar) x0
(Salimans & Ho 2022): only the first two table columns change, since every step computes x0 = c_recip z - c_recipm1 out and
the guidance (1 + w) out_c - w out_u is linear in the output.

w=None samples a model whose guidance is in its weights, such as a progressively distilled student (distill.py): one
B-batch conditional forward per step, stepped by `xunet_sampler_step_cond`.  `distill_grid` gives the timesteps such a
student was trained on, and `Schedule(timesteps=...)` the schedule of any such grid.

guide_params samples with autoguidance (Karras et al. 2024): the negative of the guidance is a weaker version of the same
model (fewer training steps, a shorter EMA, a narrower config) under the same conditioning, instead of the pose-dropped
branch.  Each step is a B-batch forward of the main model, a B-batch forward of the guide on the same device inputs, and
`xunet_sampler_step_guide`: (1 + w) out_main - w out_guide.

method='consistency' samples a consistency-distilled student (distill.ConsistencyTeacher) by multistep consistency sampling
(Song et al. 2023, Alg. 1): x0 = clip(f(z, t_k)), then z' = alpha' x0 + sigma' eps' with fresh noise, landing on x0 after
the last step.  `consistency_grid` gives its timesteps.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .xunet import XUNet, BATCH_KEYS, Engine, ParamTree, pack_flat


def cosine_beta_schedule(timesteps, s=0.008):
    """sampling.py:16-26 (float64)."""
    steps = timesteps + 1
    x = np.linspace(0, timesteps, steps, dtype=np.float64)
    ac = np.cos(((x / timesteps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = 1 - (ac[1:] / ac[:-1])
    return np.clip(betas, 0, 0.9999)


def logsnr_schedule_cosine(t, *, logsnr_min=-20., logsnr_max=20.):
    """sampling.py:73-76."""
    b = np.arctan(np.exp(-.5 * logsnr_max))
    a = np.arctan(np.exp(-.5 * logsnr_min)) - b
    return -2. * np.log(np.tan(a * t + b))


METHODS = ('ddpm', 'ddim', 'dpmpp_2m')
# every sampler method: the teacher samplers, and multistep consistency sampling of a consistency-distilled student
SAMPLER_METHODS = METHODS + ('consistency',)
SPACINGS = ('linear', 'logsnr')
PREDICTIONS = ('eps', 'v')


def check_prediction(prediction) -> str:
    """Validates what the network predicts: 'eps' (the noise) or 'v' (sqrt(abar) eps - sqrt(1 - abar) x0)."""
    if prediction not in PREDICTIONS:
        raise ValueError(f'prediction must be one of {PREDICTIONS}, got {prediction!r}')
    return prediction


class Schedule:
    """The tables of sampling.py:28-41, optionally re-spaced to `steps` < T timesteps.

    spacing='linear': `steps` timesteps evenly spaced in t (all T when steps >= T).  spacing='logsnr': `steps` points
    uniform in lambda = log(sqrt(abar) / sqrt(1 - abar)) between lambda(T-1) and lambda(0), each mapped to the timestep
    with the nearest lambda, duplicates dropped.  The last steps of the cosine schedule hold a large log-SNR jump, so this
    is the spacing multistep solvers need.  With it, len(self) -- the number of forwards a sample runs -- can be smaller
    than `steps` (9 for 10, 19 for 25, 36 for 50, 142 for 256).

    timesteps: an explicit set of timesteps in [0, T), such as a distilled student's grid (`distill_grid`), in any order
    and without duplicates; it replaces `steps` and `spacing`.  The tables are built from it exactly as from a spacing's
    timesteps, so Schedule(timesteps=Schedule(n).timesteps) has the tables of Schedule(n)."""

    def __init__(self, steps: int = 1000, T: int = 1000, spacing: str = 'linear', *, timesteps=None):
        if spacing not in SPACINGS:
            raise ValueError(f'unknown spacing {spacing!r}; expected one of {SPACINGS}')
        betas_full = cosine_beta_schedule(T)
        ac_full = np.cumprod(1. - betas_full, axis=0)
        if timesteps is not None:
            ts = np.asarray(timesteps)
            if ts.ndim != 1 or ts.size == 0 or not np.issubdtype(ts.dtype, np.integer):
                raise ValueError(f'timesteps must be a non-empty 1-D array of integers, got {timesteps!r}')
            self.timesteps = np.unique(ts.astype(np.int64))
            if len(self.timesteps) != ts.size or self.timesteps[0] < 0 or self.timesteps[-1] >= T:
                raise ValueError(f'timesteps must be distinct integers in [0, {T}), got {timesteps!r}')
            ac = ac_full[self.timesteps]
        elif spacing == 'logsnr':
            lam = 0.5 * np.log(ac_full / (1. - ac_full))
            target = np.linspace(lam[T - 1], lam[0], steps)
            self.timesteps = np.unique(np.abs(lam[None, :] - target[:, None]).argmin(1))
            ac = ac_full[self.timesteps]
        elif steps >= T:
            self.timesteps = np.arange(T)
            ac = ac_full
        else:
            self.timesteps = np.unique(np.round(np.linspace(0, T - 1, steps)).astype(int))
            ac = ac_full[self.timesteps]
        ac_prev = np.pad(ac[:-1], (1, 0), 'constant', constant_values=(1))
        betas = 1. - ac / ac_prev
        alphas = 1. - betas
        self.betas, self.alphas_cumprod, self.alphas_cumprod_prev = betas, ac, ac_prev
        self.sqrt_recip_alphas_cumprod = np.sqrt(1. / ac)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1. / ac - 1)
        self.posterior_variance = betas * (1. - ac_prev) / (1. - ac)
        self.posterior_log_variance_clipped = np.log(self.posterior_variance.clip(min=1e-20))
        self.posterior_mean_coef1 = betas * np.sqrt(ac_prev) / (1. - ac)
        self.posterior_mean_coef2 = (1. - ac_prev) * np.sqrt(alphas) / (1. - ac)
        self.T = T

    def __len__(self):
        return len(self.timesteps)


def distill_grid(teacher_steps: int, rounds: int) -> np.ndarray:
    """The timesteps, in loop order (highest t first), of a model progressively distilled `rounds` times (Salimans & Ho
    2022) from a teacher sampled with DDIM on Schedule(teacher_steps, 'linear'): round 0 is that schedule's timesteps, and
    each round keeps every other timestep of the last, G_r = G_{r-1}[0::2], so the top timestep stays and the grids nest.
    Round r halves a grid of even length; an odd one raises ValueError."""
    if isinstance(rounds, bool) or int(rounds) != rounds or rounds < 0:
        raise ValueError(f'rounds must be an integer >= 0, got {rounds!r}')
    g = Schedule(teacher_steps, spacing='linear').timesteps[::-1]
    for r in range(int(rounds)):
        if len(g) % 2:
            raise ValueError(f'round {r + 1} of {rounds} would halve a grid of odd length {len(g)} '
                             f'(teacher_steps = {teacher_steps}); use a teacher_steps divisible by 2**{rounds}')
        g = g[0::2]
    return g.copy()


def consistency_grid(teacher_steps: int, k: int) -> np.ndarray:
    """The K sampling timesteps, in loop order, of a student consistency-distilled (distill.ConsistencyTeacher) on the
    teacher grid G = distill_grid(teacher_steps, 0) of N timesteps: G[(i N) // K] for i = 0..K-1.  The top timestep is
    kept and every point is a grid position the student was trained at; K = N gives G.  Raises ValueError for
    teacher_steps < 1, K < 1 or K > N."""
    for name, v in (('teacher_steps', teacher_steps), ('k', k)):
        if isinstance(v, bool) or int(v) != v or v < 1:
            raise ValueError(f'{name} must be an integer >= 1, got {v!r}')
    g = distill_grid(int(teacher_steps), 0)
    n, k = len(g), int(k)
    if k > n:
        raise ValueError(f'k = {k} sampling steps, more than the N = {n} timesteps of the teacher grid')
    return g[(np.arange(k) * n) // k].copy()


def _check_method(method: str, eta: float) -> None:
    if method not in SAMPLER_METHODS:
        raise ValueError(f'unknown sampler method {method!r}; expected one of {SAMPLER_METHODS}')
    if not 0.0 <= eta <= 1.0:
        raise ValueError(f'eta {eta} outside [0, 1]')
    if eta != 0.0 and method != 'ddim':
        raise ValueError(f'eta {eta} is only defined for method ddim, not {method}')


def _check_dynamic_threshold(p) -> None:
    """dynamic_threshold is None (the fixed clip of x0 to [-1, 1]) or a percentile p in (0, 1]."""
    if p is None:
        return
    if isinstance(p, bool) or not isinstance(p, (int, float, np.integer, np.floating)):
        raise ValueError(f'dynamic_threshold {p!r} is not a number')
    if not 0.0 < float(p) <= 1.0:          # NaN fails the comparison too
        raise ValueError(f'dynamic_threshold {p} outside (0, 1]')


def _check_feature_cache(cache_interval, cache_level, n_levels: int) -> None:
    """cache_interval N is an integer >= 1; cache_level L an integer >= 1, and at most n_levels - 1 when N > 1 (with N = 1
    every forward is full and L is not used)."""
    for name, v in (('cache_interval', cache_interval), ('cache_level', cache_level)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise ValueError(f'{name} must be an integer >= 1, got {v!r}')
    if cache_interval > 1 and cache_level > n_levels - 1:
        raise ValueError(f'cache_level {cache_level} outside [1, {n_levels - 1}] for a {n_levels}-level model')


def feature_cache_full_steps(steps: int, cache_interval: int) -> np.ndarray:
    """The uniform feature-cache schedule: (steps,) bool, True where loop position k runs a full forward (k % N == 0, so step
    0 always does) and False where it runs a cheap one."""
    return np.arange(steps) % cache_interval == 0


def sampler_table(sched: Schedule, method: str = 'ddpm', *, eta: float = 0.0, logsnr_lag: bool | None = None,
                  prediction: str = 'eps'):
    """The device table of `sched` for `method`: (rows, logsnr_first), rows (len(sched), 8) float64 (the sampler rounds
    them to fp32 once), row k = loop position k = timestep index len-1-k = {c_recip, c_recipm1, c_x0, c_z, sigma,
    logsnr_next, c_prev, 0}; logsnr_first is the log-SNR of the first forward.  A step is
        x0 = clip(c_recip z - c_recipm1 out, -1, 1);  z' = c_x0 x0 + c_z z + c_prev x0_prev + sigma noise,
    out the (guided) network output: with prediction='eps' c_recip = sqrt(1/abar), c_recipm1 = sqrt(1/abar - 1); with
    prediction='v' c_recip = sqrt(abar), c_recipm1 = sqrt(1 - abar) (x0 = alpha z - sigma_t v).  The other columns do not
    depend on the prediction.
    With abar the row's alpha-bar, abar' the next row's (1 after the last step), alpha = sqrt(abar),
    sigma_t = sqrt(1 - abar) and lambda = log(alpha / sigma_t):
      ddpm      the posterior of sampling.py:133-151 (reads the schedule's posterior tables), c_prev = 0;
      ddim      sigma = eta sqrt((1 - abar') / (1 - abar) (1 - abar / abar')), c_z = sqrt(1 - abar' - sigma^2) / sigma_t,
                c_x0 = sqrt(abar') - c_z alpha: DDIM with eps re-derived from the clipped x0 (eta = 1: the ddpm rows);
      dpmpp_2m  h = lambda' - lambda, r = h_prev / h, g = alpha' (1 - e^-h), c_z = sigma_t' / sigma_t,
                c_x0 = g (1 + 1/(2r)), c_prev = -g / (2r), sigma = 0; the first and the last row are first order
                (c_x0 = g, c_prev = 0), so the last step, to abar' = 1, is z' = x0;
      consistency  multistep consistency sampling (Song et al. 2023, Alg. 1): c_x0 = sqrt(abar'), c_z = 0,
                sigma = sqrt(1 - abar'), c_prev = 0: z' = alpha' x0 + sigma' noise, and the last step is z' = x0.
    ddim, dpmpp_2m and consistency read only sched.timesteps and the matching leading entries of sched.alphas_cumprod.
    logsnr_lag=True: the reference's lag (sampling.py:126,151): the first forward gets -20 and row k hands the next forward
    the log-SNR of its own timestep t_k.  logsnr_lag=False: each forward gets the log-SNR of the timestep z is at,
    logsnr_cosine(t_0/1000) first and logsnr_cosine(t_{k+1}/1000) from row k (the last row's value is unused).
    None (default): True, but False for consistency, whose student was trained without the lag."""
    _check_method(method, eta)
    if logsnr_lag is None:
        logsnr_lag = method != 'consistency'
    check_prediction(prediction)
    sc = sched
    n = len(sc.timesteps)
    i = np.arange(n - 1, -1, -1)
    zero = np.zeros(n)
    c_prev = zero
    if method == 'ddpm':
        sigma = np.where(i == 0, 0.0, np.exp(0.5 * sc.posterior_log_variance_clipped[i]))     # sampling.py:142-148
        c_recip, c_recipm1 = sc.sqrt_recip_alphas_cumprod[i], sc.sqrt_recipm1_alphas_cumprod[i]
        c_x0, c_z = sc.posterior_mean_coef1[i], sc.posterior_mean_coef2[i]
    else:
        ac_all = np.asarray(sc.alphas_cumprod, dtype=np.float64)[:n]
        a, a_next = ac_all[i], np.concatenate([[1.0], ac_all[:-1]])[i]
        c_recip, c_recipm1 = np.sqrt(1. / a), np.sqrt(1. / a - 1)
        if method == 'ddim':
            sigma = eta * np.sqrt((1. - a_next) / (1. - a) * (1. - a / a_next))
            # 1 - abar' - sigma^2 = (1 - abar') ((1 - eta^2) + eta^2 abar (1 - abar') / (abar' (1 - abar))), written so that
            # it does not cancel when sigma^2 is close to 1 - abar' (eta = 1 at high t)
            keep = (1. - eta ** 2) + eta ** 2 * a * (1. - a_next) / (a_next * (1. - a))
            c_z = np.sqrt((1. - a_next) * keep) / np.sqrt(1. - a)
            c_x0 = np.sqrt(a_next) - c_z * np.sqrt(a)
        elif method == 'consistency':
            sigma, c_z, c_x0 = np.sqrt(1. - a_next), zero, np.sqrt(a_next)
        else:
            sigma = zero
            c_z = np.sqrt((1. - a_next) / (1. - a))
            with np.errstate(divide='ignore', invalid='ignore'):
                lam = 0.5 * (np.log(a) - np.log(1. - a))
                lam_next = 0.5 * (np.log(a_next) - np.log(1. - a_next))        # +inf after the last step
                h = lam_next - lam
                g = -np.sqrt(a_next) * np.expm1(-h)
                r = np.concatenate([[np.nan], h[:-1]]) / h                     # h_prev / h
                second = (np.arange(n) > 0) & (np.arange(n) < n - 1)
                c_x0 = np.where(second, g * (1. + 1. / (2. * r)), g)
                c_prev = np.where(second, -g / (2. * r), 0.0)
    if prediction == 'v':
        a = np.asarray(sc.alphas_cumprod, dtype=np.float64)[:n][i]
        c_recip, c_recipm1 = np.sqrt(a), np.sqrt(1. - a)
    t = np.asarray(sc.timesteps)[i] / 1000.0
    if logsnr_lag:
        logsnr_first, logsnr_next = -20.0, logsnr_schedule_cosine(t)
    else:
        logsnr_first, logsnr_next = float(logsnr_schedule_cosine(t[0])), logsnr_schedule_cosine(np.append(t[1:], t[-1]))
    rows = np.stack([c_recip, c_recipm1, c_x0, c_z, sigma, logsnr_next, c_prev, zero], 1)
    return rows, logsnr_first


class Sampler:
    """z, the forward's z / log-SNR inputs, the loop position, the noise seed and the coefficient table all live on the device,
    so one sampler step is the 2B-batch forward, `xunet_sampler_step_table` and pos += 1, with no host arithmetic in between.
    use_graph=True replays that step as one CUDA graph; use_graph=False issues the same calls eagerly.

    method: 'ddpm' (the reference's ancestral sampler), 'ddim' (eta in [0, 1]; 0 = deterministic), 'dpmpp_2m'
    (DPM-Solver++(2M); its step is `xunet_sampler_step_multistep`, with the previous step's x0 in a device buffer) or
    'consistency' (multistep consistency sampling of a consistency-distilled student, usually with w=None,
    prediction='v' and timesteps=consistency_grid(N, K); the same table step kernels).
    spacing: the Schedule's timestep spacing, 'logsnr' for dpmpp_2m and 'linear' otherwise by default; len(self.sched)
    is the number of forwards a sample runs.  logsnr_lag: the reference's one-step lag of the network's log-SNR input,
    on by default for ddpm with prediction='eps' only (see `sampler_table`).  With every default this is the reference
    sampler.

    prediction: 'eps' (default) reads the network output as the noise; 'v' reads it as v = sqrt(abar) eps - sqrt(1 - abar) x0,
    for a model trained with create_train_state(prediction='v').  Only the table's x0 columns change (`sampler_table`), so
    every method, dynamic thresholding and sample_views run the same kernels.  The lag defaults to off for v: it is a quirk
    of the reference's eps-trained checkpoints.

    w=None: the model is sampled without classifier-free guidance, for a model whose guidance is in its weights (a
    distilled student, `distill.py`): the engine holds B rows, all with cond_mask 1, and each step is one B-batch forward
    and `xunet_sampler_step_cond`, for every method, dynamic thresholding and sample_views.  A float w (0 included) keeps
    the guided 2B batch.  timesteps: an explicit timestep grid (`Schedule(timesteps=..)`, e.g. `distill_grid`) in place of
    `steps` and `spacing`.

    dynamic_threshold: None clips x0 to [-1, 1] (the reference).  A percentile p in (0, 1] thresholds x0 per view instead
    (Saharia et al. 2022, Imagen section 2.3): s = max(1, p-quantile of |x0| over the view), x0 <- clip(x0, -s, s) / s, for
    every method, in `xunet_sampler_step_dynamic` (the paper uses p = 0.995).  It keeps guided x0 far outside [-1, 1] (large
    w at high noise) from saturating to +-1; a view whose s is 1 gets the fixed clip's bits.

    cache_interval N, cache_level L: the feature cache (DeepCache, Ma et al. 2024; `xunet_set_feature_cache`).  Loop
    position k runs a full forward when k % N == 0 and a cheap one otherwise: the cheap forward recomputes only the
    conditioning, the input conv, the blocks of the levels below L and the head, and reads the deep feature (the output of
    the up-resampler leaving level L) from the last full forward, with that step's log-SNR and inputs.  It works with every
    method, guidance and sample_views; its effect on sample quality (PSNR / SSIM on SRN) at N > 1 has not been measured.
    N = 1 (the default) runs every forward in full and gives the bits of a sampler built without these arguments.

    guide_params, guide_model: autoguidance (Karras et al. 2024, "Guiding a diffusion model with a bad version of itself").
    guide_params is the parameter tree of a weaker guide: for example the same run's post-hoc EMA reconstructed at a short
    sigma_rel and an early snapshot (`posthoc.reconstruct`, examples/posthoc_ema_srn.py).  guide_model (an XUNet or an
    XUNetConfig; default: `model`'s config) is its architecture: any config at the same image side, a narrower `ch` for
    instance.  The guide must have been trained with the same `prediction` as the model.  It needs a float w: the main
    engine then holds B rows, all with cond_mask 1 (the w=None layout, the same `model.engine(B, S, False)`), and a second
    engine of the guide config, owned by this sampler, runs the guide's B-batch forward on the main engine's device inputs
    (z, log-SNR, view, poses, cond_mask), so sample_views and the feature cache work unchanged.  A step is the two forwards
    and `xunet_sampler_step_guide`, which forms (1 + w) out_main - w out_guide with the fp32 operations of the guided step:
    w means what it means for classifier-free guidance (Karras' guidance weight is 1 + w).  Every method,
    prediction, dynamic thresholding, explicit timesteps, sample_views and the feature cache (cache_level must exist in
    both configs) work with a guide.  w = 0 gives the bits of w=None on the main params, and so does a guide equal to the
    model at w = 1.  Two B-row forwards replace the one 2B-row forward of guidance (tools/autoguide_cost.py measures
    both)."""

    def __init__(self, model: XUNet, params, batch_size: int, img_sidelength: int, *, steps: int = 1000,
                 w: float | None = 3.0, use_graph: bool = True, method: str = 'ddpm', eta: float = 0.0,
                 spacing: str | None = None, logsnr_lag: bool | None = None, dynamic_threshold: float | None = None,
                 prediction: str = 'eps', timesteps=None, cache_interval: int = 1, cache_level: int = 1,
                 guide_params=None, guide_model=None):
        _check_method(method, eta)
        _check_dynamic_threshold(dynamic_threshold)
        _check_feature_cache(cache_interval, cache_level, len(model.config.ch_mult))
        if guide_params is None and guide_model is not None:
            raise ValueError('guide_model is given without guide_params')
        if guide_params is not None and w is None:
            raise ValueError('guide_params needs a float guidance weight w; w=None samples without guidance')
        guide_cfg = None
        if guide_params is not None:
            guide_cfg = model.config if guide_model is None else getattr(guide_model, 'config', guide_model)
            _check_feature_cache(cache_interval, cache_level, len(guide_cfg.ch_mult))
        self.cache_interval, self.cache_level = int(cache_interval), int(cache_level)
        self.prediction = check_prediction(prediction)
        self.dynamic_threshold = None if dynamic_threshold is None else float(dynamic_threshold)
        self.method, self.eta = method, float(eta)
        self.logsnr_lag = (method == 'ddpm' and prediction == 'eps') if logsnr_lag is None else bool(logsnr_lag)
        self.model, self.B, self.S = model, batch_size, img_sidelength
        self.w = None if w is None else float(w)
        self.copies = 1 if w is None or guide_params is not None else 2    # engine rows per view: [cond] or [cond ; uncond]
        self.sched = Schedule(steps, spacing=('logsnr' if method == 'dpmpp_2m' else 'linear') if spacing is None else spacing,
                              timesteps=timesteps)
        self.eng = model.engine(self.copies * batch_size, img_sidelength, False)
        self.flat = model.flat_from_tree(params, img_sidelength, self.copies * batch_size)
        self.lib = _lib.load()
        self.dev = self.eng.device
        # the guide's own engine: model.engine() would hand back the main engine for a same-config guide, and the two
        # forwards would share one workspace and one output
        self.guide_eng = None if guide_cfg is None else Engine(guide_cfg, batch_size, img_sidelength, False, self.dev)
        self.guide_flat = None if guide_cfg is None else self._guide_flat(guide_params)
        self.z = torch.zeros(batch_size, img_sidelength, img_sidelength, 3, dtype=torch.float32, device=self.dev)
        self.use_graph = use_graph
        self._tab = None            # (steps, 8) coefficient table on the device
        self._noise = None          # (steps, B*S*S*3) explicit noise on the device
        self._graphs = {}           # (static conditioning, explicit noise, cheap forward) -> the captured step
        self._pos = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self._seed_base = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self._logsnr_first = -20.0
        # dpmpp_2m: the previous step's clipped x0.  Allocated once, since the captured graphs hold its pointer; a chain's
        # first row has c_prev = 0 and overwrites it, so every chain starts with a fresh history.
        self._x0_hist = torch.empty_like(self.z) if method == 'dpmpp_2m' else None

    def _guide_flat(self, params) -> torch.Tensor:
        """The guide's flat parameter buffer, laid out by the guide engine's spec; ValueError when the tree does not match."""
        g = self.guide_eng
        if isinstance(params, ParamTree) and params.flat is not None:
            if params.spec is not None and dict(params.spec) != dict(g.spec) or params.flat.numel() != g.nparams:
                raise ValueError(f'guide_params does not match the guide config {g.cfg}')
            return params.flat
        try:
            return pack_flat(params, g.spec, g.nparams).to(self.dev)
        except KeyError as err:
            raise ValueError(f'guide_params does not match the guide config {g.cfg}: {err}') from err

    def capture(self, batch: dict) -> None:
        """Runs the first 3 steps of a sample: builds the static-conditioning state and, with use_graph, the per-step CUDA
        graph (benchmarks warm up with this instead of a full `steps`-long sample)."""
        self.sample(batch, seed=0, _max_steps=3)

    def sample(self, batch: dict, *, seed: int = 0, z_init=None, noises=None, _max_steps=None) -> torch.Tensor:
        """Generates the target view for each (source image, pose pair) in `batch` (keys as data_loader.py:102-113).
        z_init / noises (list per step, index = step position high->low) make the run reproducible against the oracle."""
        B, S, e = self.B, self.S, self.eng
        # only the source image, the two poses and K condition the sampler; z / logsnr are produced by the loop itself
        # (the reference overwrites both before the first step, sampling.py:125-126)
        src = dict(batch)
        src.setdefault('z', np.zeros((B, S, S, 3), np.float32))
        src.setdefault('logsnr', np.zeros((B,), np.float32))
        dup = {k: np.concatenate([np.asarray(src[k], dtype=np.float32)] * self.copies, axis=0) for k in BATCH_KEYS}
        mask = np.concatenate([np.ones(B, np.float32), np.zeros((self.copies - 1) * B, np.float32)])
        e.load_inputs(dup, cond_mask=mask)
        steps = self._load_schedule()
        self._start_chain(seed, z_init, noises)
        self._run(steps if _max_steps is None else min(_max_steps, steps), noises is not None, static=True)
        return self.z.clone()

    def _load_schedule(self) -> int:
        """Writes the coefficient table of `self.sched` (callers may have edited it since the last call) to the device and
        returns its number of steps.  Row k = loop position k = timestep index len-1-k (`sampler_table`)."""
        rows, self._logsnr_first = sampler_table(self.sched, self.method, eta=self.eta, logsnr_lag=self.logsnr_lag,
                                                 prediction=self.prediction)
        if self._tab is None or len(self._tab) != len(rows):
            # the captured graphs hold the table and noise pointers: reallocate (and recapture) only when the length changes
            self._tab = torch.empty(len(rows), 8, dtype=torch.float32, device=self.dev)
            self._noise = None
            self._graphs = {}
        self._tab.copy_(torch.as_tensor(rows, dtype=torch.float32))
        return len(rows)

    def _start_chain(self, seed: int, z_init, noises) -> None:
        """z <- z_init, or N(0, 1) from `seed` (sampling.py:125); the first forward's inputs z and the table's first log-SNR
        (-20 with the lag, sampling.py:126); the noise of step k: noises[k], or the hash normal of seed * 1000003 + timestep
        index."""
        B, steps, e = self.B, len(self._tab), self.eng
        if z_init is None:
            g = torch.Generator(device=self.dev).manual_seed(seed)
            self.z.copy_(torch.randn(self.z.shape, generator=g, device=self.dev))
        else:
            self.z.copy_(torch.as_tensor(np.asarray(z_init), dtype=torch.float32).to(self.dev))
        e.inp['z'][:B].copy_(self.z)
        if self.copies == 2:
            e.inp['z'][B:].copy_(self.z)
        e.inp['logsnr'].fill_(self._logsnr_first)
        self._seed_base.fill_((seed * 1000003 + steps - 1) & 0x7FFFFFFFFFFFFFFF)    # the kernel subtracts the loop position
        if noises is not None:
            if self._noise is None:
                self._noise = torch.empty(steps, self.z.numel(), dtype=torch.float32, device=self.dev)
            self._noise.copy_(torch.as_tensor(np.asarray(noises[:steps]), dtype=torch.float32).reshape(steps, self.z.numel()))

    def _run(self, steps: int, noise: bool, static: bool, set_view=None) -> None:
        """The sampling loop from loop position 0: per step set_view(k) (if given), the forward, the table step and pos += 1.
        Step 0 runs eagerly, so every kernel has run once before a graph is captured.  static: poses, K, cond_mask and
        params stay fixed, so after step 0 the forwards reuse its rays, pose embeddings and weight shadows.  Steps the
        feature-cache schedule marks cheap run at cache_level (`feature_cache_full_steps`).  Both settings apply to the
        guide engine too."""
        hs = [self.eng.h] + ([] if self.guide_eng is None else [self.guide_eng.h])
        self._pos.zero_()
        full = feature_cache_full_steps(steps, self.cache_interval)
        level = 0
        try:
            for h in hs:
                self.lib.xunet_set_static_conditioning(h, 0)
            for k in range(steps):
                if set_view is not None:
                    set_view(k)
                want = 0 if full[k] else self.cache_level
                if want != level:
                    level = want
                    for h in hs:
                        _lib.check(self.lib.xunet_set_feature_cache(h, level), 'set_feature_cache')
                if k > 0 and self.use_graph:
                    self._graph(static, noise, level > 0).replay()
                else:
                    self._step(noise)
                if static and k == 0:
                    for h in hs:
                        self.lib.xunet_set_static_conditioning(h, 1)
        finally:
            # a failure mid-loop must not leave the shared engine reusing stale pose embeddings / weight shadows, or cheap
            for h in hs:
                self.lib.xunet_set_static_conditioning(h, 0)
                self.lib.xunet_set_feature_cache(h, 0)

    def _step(self, noise: bool) -> None:
        e = self.eng
        e.forward(self.flat, train=False)
        st = torch.cuda.current_stream(self.dev).cuda_stream
        hist = None if self._x0_hist is None else self._x0_hist.data_ptr()
        if self.guide_eng is not None:
            g = self.guide_eng
            g.forward(self.guide_flat, train=False, batch=e.cbatch)        # the main engine's z, log-SNR, view and poses
            _lib.check(self.lib.xunet_sampler_step_guide(e.eps.data_ptr(), g.eps.data_ptr(), self.z.data_ptr(),
                                                         self._noise.data_ptr() if noise else None, self.z.numel(), self.w,
                                                         self._tab.data_ptr(), self._pos.data_ptr(), self._seed_base.data_ptr(),
                                                         hist, self.B, self.dynamic_threshold or 0.0, None,
                                                         e.inp['z'].data_ptr(), e.inp['logsnr'].data_ptr(), st),
                       'sampler_step_guide')
            self._pos.add_(1)
            return
        if self.w is None:
            _lib.check(self.lib.xunet_sampler_step_cond(e.eps.data_ptr(), self.z.data_ptr(),
                                                        self._noise.data_ptr() if noise else None, self.z.numel(),
                                                        self._tab.data_ptr(), self._pos.data_ptr(), self._seed_base.data_ptr(),
                                                        hist, self.B, self.dynamic_threshold or 0.0, None,
                                                        e.inp['z'].data_ptr(), e.inp['logsnr'].data_ptr(), st),
                       'sampler_step_cond')
            self._pos.add_(1)
            return
        head = (e.eps.data_ptr(), self.z.data_ptr(), self._noise.data_ptr() if noise else None, self.z.numel(), self.w,
                self._tab.data_ptr(), self._pos.data_ptr(), self._seed_base.data_ptr())
        tail = (e.inp['z'].data_ptr(), e.inp['logsnr'].data_ptr(), 2 * self.B, st)
        if self.dynamic_threshold is not None:
            _lib.check(self.lib.xunet_sampler_step_dynamic(*head, hist, self.B, self.dynamic_threshold, None, *tail),
                       'sampler_step_dynamic')
        elif self._x0_hist is None:
            _lib.check(self.lib.xunet_sampler_step_table(*head, *tail), 'sampler_step_table')
        else:
            _lib.check(self.lib.xunet_sampler_step_multistep(*head, self._x0_hist.data_ptr(), *tail), 'sampler_step_multistep')
        self._pos.add_(1)

    def _graph(self, static: bool, noise: bool, cheap: bool) -> torch.cuda.CUDAGraph:
        """The captured step; static conditioning, explicit noise and a cheap forward each change what it launches."""
        key = (static, noise, cheap)
        if key not in self._graphs:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.Stream(device=self.dev)):
                self._step(noise)
            self._graphs[key] = g
        return self._graphs[key]

    # ---- stochastic conditioning (3DiM, Watson et al. 2022, section 3.2; the reference implements only k = 1) ---------
    def sample_views(self, views, poses, K, target_poses, *, seed: int = 0, condition_on_generated: bool = True,
                     return_choices: bool = False, z_init=None, noises=None):
        """Autoregressive multi-view generation with STOCHASTIC CONDITIONING.

        views  : (B, k, S, S, 3) known source images in [-1, 1];  poses: dict R (B, k, 3, 3), t (B, k, 3) of those views
        K      : (B, 3, 3) intrinsics;  target_poses: dict R (B, m, 3, 3), t (B, m, 3)
        For each of the m target poses in turn the chain starts from noise and, at EVERY denoising step, conditions on
        one view drawn uniformly from the pool (the k sources plus -- if condition_on_generated -- the targets generated
        so far), exactly as the paper's sampler; one 2B-batch forward per step ([cond ; uncond], guidance weight w) and
        the same posterior update as `sample()` (w=None: one B-batch conditional forward; with a guide: the main and the
        guide B-batch forwards, the guide reading the main engine's inputs).  The pool lives on the device; a step only copies the chosen view and
        its pose into the engine's input buffers before the step, which runs with the full forward (static conditioning
        off).  z_init (m, B,S,S,3) / noises (m, steps, B,S,S,3) make a run reproducible against the oracle; with one
        source, one target and the same seed the result equals `sample()`.  With a feature cache (cache_interval > 1) a view
        is drawn on full steps only: a cheap step keeps the view of the last full step, which its cached deep feature saw.
        Returns (B, m, S, S, 3) [and the (m, steps) pool indices in use at each step]."""
        B, e = self.B, self.eng
        dev = self.dev
        f32 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32).to(dev)
        pool_x = [v for v in f32(views).unbind(1)]                     # each (B,S,S,3)
        pool_R = [v for v in f32(poses['R']).unbind(1)]
        pool_t = [v for v in f32(poses['t']).unbind(1)]
        tR, tt = f32(target_poses['R']), f32(target_poses['t'])
        m = tR.shape[1]
        Kd = f32(K)
        rng = np.random.RandomState(seed)
        steps = self._load_schedule()
        full = feature_cache_full_steps(steps, self.cache_interval)
        cp = self.copies
        e.inp['K'].copy_(torch.cat([Kd] * cp, 0).reshape(e.inp['K'].shape))
        e.inp['cond_mask'].copy_(torch.cat([torch.ones(B, device=dev), torch.zeros((cp - 1) * B, device=dev)]))
        outs, choices = [], []
        for j in range(m):
            e.inp['R2'].copy_(torch.cat([tR[:, j]] * cp, 0).reshape(e.inp['R2'].shape))
            e.inp['t2'].copy_(torch.cat([tt[:, j]] * cp, 0).reshape(e.inp['t2'].shape))
            self._start_chain(seed + 7919 * j, None if z_init is None else z_init[j], None if noises is None else noises[j])
            row = []

            def set_view(k):
                if not full[k]:
                    row.append(row[-1])
                    return
                c = int(rng.randint(len(pool_x)))
                row.append(c)
                e.inp['x'].copy_(torch.cat([pool_x[c]] * cp, 0).reshape(e.inp['x'].shape))
                e.inp['R1'].copy_(torch.cat([pool_R[c]] * cp, 0).reshape(e.inp['R1'].shape))
                e.inp['t1'].copy_(torch.cat([pool_t[c]] * cp, 0).reshape(e.inp['t1'].shape))

            self._run(steps, noises is not None, static=False, set_view=set_view)
            out = self.z.clone()
            outs.append(out)
            choices.append(row)
            if condition_on_generated:
                pool_x.append(out); pool_R.append(tR[:, j]); pool_t.append(tt[:, j])
        res = torch.stack(outs, 1)
        return (res, np.asarray(choices)) if return_choices else res


def save_view(path: str, img) -> None:
    """Writes an image in [-1,1] (HWC, RGB) as PNG: the headless replacement of cv2.imshow(z/2+0.5) (sampling.py:153)."""
    import cv2
    a = np.clip(np.asarray(img, dtype=np.float32) / 2.0 + 0.5, 0.0, 1.0)
    cv2.imwrite(path, (a[:, :, ::-1] * 255.0 + 0.5).astype(np.uint8))
