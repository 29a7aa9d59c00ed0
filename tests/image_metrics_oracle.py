"""The CPU restatement of the reference evaluation script's image metrics (scripts/eval.py: skimage's peak_signal_noise_ratio and
rgb_ssim on 8-bit images), in float64 numpy / scipy, for the tests.  Test infrastructure: never imported by the f2nerf_b200
package.  tests/golden/ref_eval_metrics.npz holds the script's own values for seeded image pairs (oracle/make_golden_metrics.py).
"""
import numpy as np
import scipy.signal


def pred_to_u8(x):
    """A rendered image as TestImages writes it: Utils::WriteImageTensor's (x * 255).clip(0, 255).to(uint8) in fp32, i.e.
    trunc(clip(x, 0, 1) * 255)."""
    return np.trunc(np.clip(np.asarray(x, np.float32), 0., 1.) * np.float32(255.)).astype(np.uint8)


def gt_to_u8(x):
    """A ground-truth image in [0, 1] as its stored byte: rint(clip(x, 0, 1) * 255) in fp32 (exact for u8 / 255.f)."""
    return np.rint(np.clip(np.asarray(x, np.float32), 0., 1.) * np.float32(255.)).astype(np.uint8)


def sse(a_u8, b_u8):
    """The exact integer sum of squared differences of two uint8 images."""
    d = a_u8.astype(np.int64) - b_u8.astype(np.int64)
    return int((d * d).sum())


def psnr(a_u8, b_u8):
    """peak_signal_noise_ratio(a, b) for uint8 images: 10 log10(255^2 / MSE), the MSE a float64 mean; inf when a == b."""
    e = sse(a_u8, b_u8)
    if e == 0:
        return float("inf")
    return float(10. * np.log10(65025. / (np.float64(e) / np.float64(a_u8.size))))


def gaussian_taps(size=11, sigma=1.5):
    """Normalised 1D Gaussian of ``size`` taps centred on the middle one."""
    k = np.arange(size) - size // 2
    f = np.exp(-0.5 * (k / sigma) ** 2)
    return f / f.sum()


def ssim_map(a_u8, b_u8, size=11, sigma=1.5, k1=0.01, k2=0.03):
    """The mip-NeRF SSIM map of two uint8 [H,W,3] images scaled to [0, 1] (float64): per channel a separable 'valid' Gaussian
    blur of x, y, x^2, y^2, xy, variances clipped at 0, the covariance's magnitude clipped to sqrt(var_x var_y)
    -> [H-size+1, W-size+1, 3]."""
    x, y = a_u8.astype(np.float64) / 255., b_u8.astype(np.float64) / 255.
    f = gaussian_taps(size, sigma)

    def blur(z):
        return np.stack([scipy.signal.convolve2d(scipy.signal.convolve2d(z[..., c], f[:, None], mode="valid"), f[None, :],
                                                 mode="valid") for c in range(z.shape[-1])], -1)

    mx, my = blur(x), blur(y)
    vx = np.maximum(blur(x * x) - mx * mx, 0.)
    vy = np.maximum(blur(y * y) - my * my, 0.)
    cxy = blur(x * y) - mx * my
    cxy = np.sign(cxy) * np.minimum(np.sqrt(vx * vy), np.abs(cxy))
    c1, c2 = k1 ** 2, k2 ** 2
    return (2. * mx * my + c1) * (2. * cxy + c2) / ((mx * mx + my * my + c1) * (vx + vy + c2))


def ssim(a_u8, b_u8):
    """Mean of ``ssim_map`` over all pixels and channels."""
    return float(np.mean(ssim_map(a_u8, b_u8)))
