"""TEST INFRASTRUCTURE — numpy restatement of the full-reference scores the reference's test configuration asks for,
used only by tests/ and tools/ as the checker for the device scores (pgt_frame_scores, pgtformer_b200/metrics.py).
Not a product path.

`options/release_test_stage_IIII_dont_need_align_version.yml` (val.metrics) scores restored frames with basicsr's
`calculate_psnr` and `calculate_ssim`, `crop_border: 0`, `test_y_channel: false`.  basicsr is neither installed nor part
of the reference tree, so this module restates what basicsr 1.4 computes with those settings, in float64, for rgb24
frames a, b of shape [H, W, 3] uint8:

    PSNR:  mse = mean((a - b)^2) over all H W 3 values; 10 log10(255^2 / mse), inf when mse == 0.
    SSIM:  per channel, with the 11 x 11 window outer(k, k), k = cv2.getGaussianKernel(11, 1.5)
           (exp(-(i - 5)^2 / (2 1.5^2)) normalised to sum 1), and filter() over the valid region only (output pixel
           (i, j) for i in [5, H - 5), j in [5, W - 5)):
               mu1 = filter(x), mu2 = filter(y), sigma1^2 = filter(x^2) - mu1^2, sigma2^2 = filter(y^2) - mu2^2,
               sigma12 = filter(x y) - mu1 mu2,
               map = ((2 mu1 mu2 + C1)(2 sigma12 + C2)) / ((mu1^2 + mu2^2 + C1)(sigma1^2 + sigma2^2 + C2)),
               C1 = (0.01 255)^2, C2 = (0.03 255)^2;
           the channel's score is the map's mean and the frame's the mean of its three channels.

basicsr computes filter() as `cv2.filter2D(img, -1, window)[5:-5, 5:-5]`, which OpenCV runs through a DFT for an
11 x 11 float64 kernel.  `ssim_channels` sums the window directly as two separable passes (horizontal, then vertical),
which needs no cv2; `ssim_channels_cv2` is basicsr's form, available where cv2 imports.  Frames smaller than 11 x 11
raise ValueError (basicsr returns NaN with a warning).  Both scores are invariant to channel order, so BGR and RGB
frames score the same.
"""
import numpy as np

R = 5                                    # window radius: 11 taps
C1 = (0.01 * 255) ** 2
C2 = (0.03 * 255) ** 2


def gaussian_window():
    """The 11 taps cv2.getGaussianKernel(11, 1.5) returns, float64."""
    i = np.arange(2 * R + 1, dtype=np.float64)
    k = np.exp(-(i - R) ** 2 / (2 * 1.5 ** 2))
    return k / k.sum()


def _check(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.ndim != 3 or a.shape[-1] != 3 or a.dtype != np.uint8 or b.dtype != np.uint8:
        raise ValueError('expected two rgb24 frames [H,W,3] uint8 of one shape, got %s %s and %s %s'
                         % (a.shape, a.dtype, b.shape, b.dtype))
    if a.shape[0] < 2 * R + 1 or a.shape[1] < 2 * R + 1:
        raise ValueError('SSIM needs frames of at least 11 x 11, got %dx%d' % a.shape[:2])
    return a, b


def sse(a, b):
    """The exact integer sum of squared differences over all H W 3 values."""
    a, b = _check(a, b)
    d = a.astype(np.int64) - b.astype(np.int64)
    return int((d * d).sum())


def psnr(a, b):
    """basicsr's calculate_psnr(a, b, crop_border=0, test_y_channel=False): a float64 value, or inf."""
    a, b = _check(a, b)
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    if mse == 0:
        return float('inf')
    return 10. * np.log10(255. * 255. / mse)


def _map_mean(mu1, mu2, fxx, fyy, fxy):
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    sigma1_sq, sigma2_sq, sigma12 = fxx - mu1_sq, fyy - mu2_sq, fxy - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    return ssim_map.mean()


def _filter_valid(img, k):
    """The 11 x 11 window outer(k, k) summed directly at every output pixel of the valid region: [H - 10, W - 10]."""
    H, W = img.shape
    h = sum(k[q] * img[:, q:q + W - 2 * R] for q in range(2 * R + 1))
    return sum(k[q] * h[q:q + H - 2 * R] for q in range(2 * R + 1))


def ssim_channels(a, b):
    """Each channel's SSIM, float64 [3], with the window summed directly."""
    a, b = _check(a, b)
    k = gaussian_window()
    out = []
    for c in range(3):
        x, y = a[..., c].astype(np.float64), b[..., c].astype(np.float64)
        out.append(_map_mean(*(_filter_valid(t, k) for t in (x, y, x * x, y * y, x * y))))
    return np.array(out)


def ssim_channels_cv2(a, b):
    """Each channel's SSIM, float64 [3], as basicsr computes it with cv2.filter2D (needs cv2)."""
    import cv2
    a, b = _check(a, b)
    kernel = cv2.getGaussianKernel(11, 1.5)
    window = np.outer(kernel, kernel.transpose())
    out = []
    for c in range(3):
        x, y = a[..., c].astype(np.float64), b[..., c].astype(np.float64)
        out.append(_map_mean(*(cv2.filter2D(t, -1, window)[R:-R, R:-R] for t in (x, y, x ** 2, y ** 2, x * y))))
    return np.array(out)


def ssim(a, b, cv2_form=False):
    """basicsr's calculate_ssim(a, b, crop_border=0, test_y_channel=False): the mean of the three channel values."""
    return np.array(list((ssim_channels_cv2 if cv2_form else ssim_channels)(a, b))).mean()


def score(restored, gt, cv2_form=False):
    """{'psnr': float64 [N], 'ssim': float64 [N]} of N frame pairs [N, H, W, 3] uint8, frame by frame."""
    restored, gt = np.asarray(restored), np.asarray(gt)
    return {'psnr': np.array([psnr(a, b) for a, b in zip(restored, gt)], np.float64),
            'ssim': np.array([ssim(a, b, cv2_form) for a, b in zip(restored, gt)], np.float64)}
