"""float64 reference of the image metrics of xunet_image_metrics (include/xunet_b200.h), restating
skimage.metrics.structural_similarity(u_pred, u_target, channel_axis=-1, data_range=1, gaussian_weights=True, sigma=1.5,
use_sample_covariance=False): each channel is filtered with scipy's Gaussian (sigma 1.5, truncate 3.5 -> 11 taps, reflect
padding), the 5-pixel border whose windows reach the padding is cropped, and the SSIM map is averaged.  Also MSE / PSNR with
data range 1.  Inputs are (B,S,S,3) in [-1, 1]; values are mapped to u = clamp((v + 1) / 2, 0, 1) first."""
import numpy as np
from scipy.ndimage import gaussian_filter

C1, C2 = 0.01 ** 2, 0.03 ** 2
SIGMA, TRUNCATE, PAD = 1.5, 3.5, 5


def to_unit(v) -> np.ndarray:
    return np.clip((np.asarray(v, dtype=np.float64) + 1.0) / 2.0, 0.0, 1.0)


def ssim_from_moments(mp, mt, pp, tt, pt):
    vp, vt, cpt = pp - mp * mp, tt - mt * mt, pt - mp * mt
    return (2 * mp * mt + C1) * (2 * cpt + C2) / ((mp * mp + mt * mt + C1) * (vp + vt + C2))


def ssim(pred, target) -> np.ndarray:
    """(B,) SSIM per image."""
    up, ut = to_unit(pred), to_unit(target)
    out = []
    for p_img, t_img in zip(up, ut):
        vals = []
        for c in range(3):
            p, t = p_img[..., c], t_img[..., c]
            f = lambda a: gaussian_filter(a, sigma=SIGMA, truncate=TRUNCATE, mode='reflect')[PAD:-PAD, PAD:-PAD]
            vals.append(ssim_from_moments(f(p), f(t), f(p * p), f(t * t), f(p * t)))
        out.append(np.mean(vals))
    return np.asarray(out)


def mse_psnr(pred, target):
    """(B,) MSE and (B,) PSNR in dB (+inf for identical images)."""
    d = to_unit(pred) - to_unit(target)
    mse = (d * d).reshape(len(d), -1).mean(1)
    with np.errstate(divide='ignore'):
        return mse, -10.0 * np.log10(mse)


PAIR_KINDS = ('noise', 'smooth', 'srn', 'near_white', 'identical')


def make_pair(kind: str, B: int, S: int, seed: int = 0):
    """(pred, target), each (B,S,S,3) float32 in [-1, 1] (up to deliberate clipping):
    noise       independent uniform noise;
    smooth      a smooth random field against itself plus N(0, 0.01) noise;
    srn         a white background with a shaded coloured blob against the same scene shifted by a few pixels;
    near_white  u = 0.98 + N(0, 0.001) for both, independently (the cancellation case of sigma^2 = E[u^2] - mu^2);
    identical   one random image twice."""
    rng = np.random.RandomState(seed)
    shape = (B, S, S, 3)
    if kind == 'noise':
        p, t = rng.uniform(-1, 1, shape), rng.uniform(-1, 1, shape)
    elif kind == 'smooth':
        f = np.stack([gaussian_filter(rng.randn(S, S, 3), sigma=(S / 8, S / 8, 0), mode='wrap') for _ in range(B)])
        t = np.tanh(f / f.std())
        p = np.clip(t + 0.01 * rng.randn(*shape), -1, 1)
    elif kind == 'srn':
        yy, xx = np.mgrid[0:S, 0:S] / S
        imgs = []
        for _ in range(B):
            cy, cx, r = rng.uniform(0.35, 0.65), rng.uniform(0.35, 0.65), rng.uniform(0.15, 0.3)
            inside = ((yy - cy) ** 2 + (xx - cx) ** 2 < r * r)[..., None]
            blob = rng.uniform(-0.8, 0.4, 3) + 0.3 * (yy - cy)[..., None] + 0.02 * rng.randn(S, S, 3)
            imgs.append(np.where(inside, blob, 1.0))
        t = np.stack(imgs)
        p = np.roll(t, shift=(rng.randint(1, 4), rng.randint(-3, 4)), axis=(1, 2))
    elif kind == 'near_white':
        p = 2 * (0.98 + 0.001 * rng.randn(*shape)) - 1
        t = 2 * (0.98 + 0.001 * rng.randn(*shape)) - 1
    elif kind == 'identical':
        t = rng.uniform(-1, 1, shape)
        p = t
    else:
        raise ValueError(kind)
    return p.astype(np.float32), np.array(t, dtype=np.float32)
