"""Full-reference scores of restored frames on the device: PSNR and SSIM as the reference's test configuration defines
them (`options/release_test_stage_IIII_dont_need_align_version.yml`, val.metrics: basicsr's `calculate_psnr` and
`calculate_ssim`, `crop_border: 0`, `test_y_channel: false`, over the rgb frame; restated in oracle/metrics_oracle.py).

The device (pgt_frame_scores) returns each frame's exact integer sum of squared differences and each channel's SSIM map
mean in fp64.  PSNR is formed here from that exact sum with basicsr's own numpy expression, so it is bit for bit what
basicsr gives; SSIM agrees with it to about 1e-15 (the window sums run in another order).
`VideoRestorer.evaluate` scores inside its batch loop, on the restored frames before they leave the device.
"""
import numpy as np
import torch

from . import ops

MIN_SIDE = 11                            # the SSIM window


def check_frames(x, name):
    """rgb24 frames [N,H,W,3] uint8 with H, W >= 11 (numpy, or a host or CUDA torch tensor), checked on the host; ->
    a torch tensor sharing x's memory where it can.  Anything else raises ValueError."""
    if torch.is_tensor(x):
        t = x
    else:
        a = np.asarray(x)
        if a.dtype != np.uint8:
            raise ValueError('%s: expected rgb24 frames [N,H,W,3] uint8, got %s %s' % (name, a.shape, a.dtype))
        t = torch.from_numpy(np.ascontiguousarray(a))
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError('%s: expected rgb24 frames [N,H,W,3] uint8, got %s %s' % (name, tuple(t.shape), t.dtype))
    if t.shape[1] < MIN_SIDE or t.shape[2] < MIN_SIDE:
        raise ValueError('%s: SSIM needs frames of at least %d x %d, got %dx%d'
                         % (name, MIN_SIDE, MIN_SIDE, t.shape[1], t.shape[2]))
    return t


def finish(sse, ssim, hw):
    """{'psnr': float64 [N], 'ssim': float64 [N]} from the device's sse [N] (exact integers) and per-channel SSIM
    [N, 3] of frames of hw = (H, W), with basicsr's expressions: mse = sse / (H W 3) is what np.mean of the squared
    differences gives, since their float64 sum is exact."""
    n = hw[0] * hw[1] * 3
    psnr = []
    for s in np.asarray(sse, np.int64):
        mse = np.float64(s) / n
        psnr.append(float('inf') if mse == 0 else 10. * np.log10(255. * 255. / mse))
    return {'psnr': np.array(psnr, np.float64).reshape(-1),
            'ssim': np.array([np.array(list(c)).mean() for c in np.asarray(ssim, np.float64)], np.float64).reshape(-1)}


def _on(t, dev):
    if t.is_cuda:
        return t.contiguous()
    return t.contiguous().pin_memory().to(dev, non_blocking=True)


@torch.no_grad()
def score(restored, gt):
    """PSNR and SSIM of each pair of rgb24 frames restored[i], gt[i]: uint8 [N,H,W,3], H, W >= 11, numpy or host or
    CUDA torch tensors.  -> {'psnr': float64 [N], 'ssim': float64 [N]} as numpy arrays (psnr inf for identical
    frames).  Shapes and dtypes are checked before any device work; host frames cross to the device through pinned
    memory, on the device of a CUDA input (the current device when both are on the host)."""
    a, b = check_frames(restored, 'restored'), check_frames(gt, 'gt')
    if a.shape != b.shape:
        raise ValueError('restored %s and gt %s differ in shape' % (tuple(a.shape), tuple(b.shape)))
    if a.is_cuda and b.is_cuda and a.device != b.device:
        raise ValueError('restored and gt are on different devices: %s, %s' % (a.device, b.device))
    hw = (int(a.shape[1]), int(a.shape[2]))
    if a.shape[0] == 0:
        return finish(np.zeros(0, np.int64), np.zeros((0, 3)), hw)
    dev = a.device if a.is_cuda else b.device if b.is_cuda else torch.device('cuda', torch.cuda.current_device())
    with torch.cuda.device(dev):
        sse, ssim = ops.frame_scores(_on(a, dev), _on(b, dev))
        return finish(sse.cpu().numpy(), ssim.cpu().numpy(), hw)
