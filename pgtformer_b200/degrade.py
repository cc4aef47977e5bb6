"""The `lr` degradation of the reference's test set, on the device (`data/vfhq_full_dataset.py:983-988,1017-1024`):
each ground-truth frame is downscaled with basicsr's antialiased bicubic imresize (`basicsr/utils/matlab_functions.py`,
basicsr 1.4) of `v / 255.0` in float32, and `Engine.restore_windows(downscale=...)` then upsamples the fp32 result
with F.interpolate(mode='bilinear', align_corners=True) to the model's size.  The low-resolution frames stay fp32,
unclamped: bicubic overshoot below 0 and above 1 reaches the model.

This module is the only builder and reader of the tap tables pgt_imresize_u8hwc_to_f32nchw takes: per axis, fp32
weights [out, K] computed with basicsr's own torch float32 expressions (calculate_weights_indices, cubic), and int32
indices [out, K] of the source samples they weigh, with basicsr's symmetric padding (the edge sample repeated)
already folded into [0, in), so the kernel has no padding logic.  Tables are built on the host, uploaded once per
(device, in_len, out_len, scale) and never allocated inside a CUDA graph capture.

Each pass is defined as the fp32 value nearest to the exact sum of its fp32 products w * x (ties to even), which no
summation order changes; basicsr's `mv` sums in its BLAS's order and agrees with it to a few ulps.  The kernel sums
exactly as long as the accumulated rounding errors of a double-double stay below 2^53 times the products' common
quantum; `plan` checks that bound for every table and rejects a scale whose taps break it (DESIGN.md §6d).  Scales
1/2, 1/3 and 1/4 pass at every frame size.
"""
import functools
import math

import numpy as np
import torch

from . import ops


def _cubic(x):
    """basicsr's cubic: Keys' kernel with a = -0.5, in its piecewise form."""
    absx = torch.abs(x)
    absx2 = absx ** 2
    absx3 = absx ** 3
    return (1.5 * absx3 - 2.5 * absx2 + 1) * ((absx <= 1).type_as(absx)) + \
        (-0.5 * absx3 + 2.5 * absx2 - 4 * absx + 2) * (((absx > 1) * (absx <= 2)).type_as(absx))


def _weights_indices(in_len, out_len, scale):
    """basicsr's calculate_weights_indices(in_len, out_len, scale, 'cubic', 4, antialiasing=True) for scale < 1:
    (weights fp32 [out, K], 1-based first-tap positions in the padded axis [out, K] int64, sym_len_s, sym_len_e)."""
    kernel_width = 4 / scale
    x = torch.linspace(1, out_len, out_len)
    u = x / scale + 0.5 * (1 - 1 / scale)
    left = torch.floor(u - kernel_width / 2)
    p = math.ceil(kernel_width) + 2
    indices = left.view(out_len, 1).expand(out_len, p) + torch.linspace(0, p - 1, p).view(1, p).expand(out_len, p)
    distance_to_center = u.view(out_len, 1).expand(out_len, p) - indices
    weights = scale * _cubic(distance_to_center * scale)
    weights_sum = torch.sum(weights, 1).view(out_len, 1)
    weights = weights / weights_sum.expand(out_len, p)
    weights_zero_tmp = torch.sum((weights == 0), 0)
    if not math.isclose(weights_zero_tmp[0], 0, rel_tol=1e-6):
        indices = indices.narrow(1, 1, p - 2)
        weights = weights.narrow(1, 1, p - 2)
    if not math.isclose(weights_zero_tmp[-1], 0, rel_tol=1e-6):
        indices = indices.narrow(1, 0, p - 2)
        weights = weights.narrow(1, 0, p - 2)
    weights = weights.contiguous()
    indices = indices.contiguous()
    sym_len_s = -indices.min() + 1
    sym_len_e = indices.max() - in_len
    indices = indices + sym_len_s - 1
    return weights, indices.long(), int(sym_len_s), int(sym_len_e)


def _low_bit(w):
    """The exponent of the lowest set bit of each nonzero fp32 value in w (numpy), as an int64 array."""
    w = np.asarray(w, np.float32).reshape(-1)
    w = w[w != 0]
    bits = w.view(np.int32).astype(np.int64)
    e = (bits >> 23) & 0xff
    m = np.where(e > 0, (bits & 0x7fffff) | 0x800000, bits & 0x7fffff)
    tz = np.zeros_like(m)
    while (m & 1 == 0).any():
        step = (m & 1) == 0
        tz += step
        m = np.where(step, m >> 1, m)
    return np.maximum(e, 1) - 150 + tz


@functools.lru_cache(maxsize=None)
def taps(in_len, scale):
    """One axis of in_len samples downscaled by `scale` (0 < scale < 1): (weights fp32 [out, K], indices int32
    [out, K] into [0, in_len), low-bit exponent of the weights, max row sum of |w|) on the host.  ValueError where
    basicsr's imresize cannot run (its symmetric padding must fit inside the axis)."""
    out_len = math.ceil(in_len * scale)
    if out_len < 1:
        raise ValueError('imresize by %r of %d samples gives no output' % (scale, in_len))
    weights, indices, sym_s, sym_e = _weights_indices(in_len, out_len, scale)
    if not (0 <= sym_s <= in_len and 1 <= sym_e <= in_len):
        raise ValueError('imresize by %r needs a side of at least %d samples for its symmetric padding, got %d'
                         % (scale, max(sym_s, sym_e), in_len))
    # padded position a -> source sample: a < s mirrors the first s samples, a >= s + in the last e (edge repeated)
    q = indices - sym_s
    src = torch.where(q < 0, -q - 1, torch.where(q >= in_len, 2 * in_len - q - 1, q))
    w64 = weights.double()
    return weights, src.to(torch.int32), int(_low_bit(weights.numpy()).min()), float(w64.abs().sum(1).max())


def check_scale(scale):
    """A downscale factor from the caller as a float in (0, 1); else ValueError."""
    try:
        s = float(scale)
    except (TypeError, ValueError):
        raise ValueError('downscale must be a number, got %r' % (scale,)) from None
    if not (0 < s < 1):
        raise ValueError('downscale must be in (0, 1), got %r' % (scale,))
    return s


def plan(hw, scale):
    """The tap tables of frames hw = (h, w) downscaled by `scale` -> (taps of H, taps of W), checked on the host:
    0 < scale < 1, basicsr's padding fits both sides, and the exact-sum bound of DESIGN.md §6d holds for both passes
    (pass 1 sums fp32 weights times x = (float)(v / 255.0), multiples of 2^-31 at most 1; pass 2 sums the other
    axis's weights times pass 1's outputs, multiples of pass 1's quantum).  Anything else raises ValueError."""
    scale = check_scale(scale)
    h, w = (int(v) for v in hw)
    if h < 1 or w < 1:
        raise ValueError('downscale needs frames of at least 1 x 1, got %dx%d' % (h, w))
    th, tw = taps(h, scale), taps(w, scale)
    (wh, _, qh, ah), (ww, _, qw, aw) = th, tw
    kh, kw = wh.shape[1], ww.shape[1]
    if math.log2(kh * ah) > 74 + qh or math.log2(kw * aw * ah * (1 + 2.0 ** -23)) > 74 + qh + qw:
        raise ValueError('downscale %r: its bicubic taps are too fine for the device to sum exactly' % (scale,))
    return th, tw


def out_size(hw, scale):
    """(ceil(h scale), ceil(w scale)), basicsr's output size."""
    return math.ceil(int(hw[0]) * float(scale)), math.ceil(int(hw[1]) * float(scale))


_device_taps = {}


def _on_device(t, dev, key):
    """The (weights, indices) of host taps t on dev, uploaded once per key; never inside a graph capture."""
    got = _device_taps.get(key)
    if got is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('imresize tap tables must be uploaded before a CUDA graph capture')
        got = _device_taps[key] = (t[0].to(dev), t[1].to(dev))
    return got


def resize(frames_u8, scale, out):
    """Device work: rgb24 frames [F,h,w,3] uint8 on the device -> out fp32 [F,3,*out_size] (plan must accept the
    arguments; callers check them first)."""
    F, h, w, _ = frames_u8.shape
    th, tw = plan((h, w), scale)
    dev, s = frames_u8.device, float(scale)
    oh, ow = out_size((h, w), s)
    return ops.imresize_u8hwc_to_f32nchw(frames_u8, _on_device(th, dev, (dev, h, oh, s)),
                                         _on_device(tw, dev, (dev, w, ow, s)), out)


@torch.no_grad()
def downsample(frames_u8, scale=0.25):
    """The `lr` branch's low-resolution frames: rgb24 frames [N,h,w,3] uint8 (numpy, or a host or CUDA torch tensor)
    -> fp32 CUDA tensor [N,3,ceil(h scale),ceil(w scale)], basicsr's imresize of v / 255.0, not clamped.  On the
    device of a CUDA input, else the current device.  Arguments are checked before any device work (ValueError)."""
    t = frames_u8 if torch.is_tensor(frames_u8) else np.asarray(frames_u8)
    u8 = t.dtype == (torch.uint8 if torch.is_tensor(t) else np.uint8)
    if not u8 or t.ndim != 4 or t.shape[-1] != 3:
        raise ValueError('expected rgb24 frames [N,H,W,3] uint8, got %s %s' % (tuple(t.shape), t.dtype))
    n, h, w = (int(v) for v in t.shape[:3])
    plan((h, w), scale)
    oh, ow = out_size((h, w), scale)
    dev = t.device if torch.is_tensor(t) and t.is_cuda else torch.device('cuda', torch.cuda.current_device())
    with torch.cuda.device(dev):
        out = torch.empty(n, 3, oh, ow, dtype=torch.float32, device=dev)
        if n == 0:
            return out
        if torch.is_tensor(t) and t.is_cuda:
            x = t.contiguous()
        else:
            x = (t if torch.is_tensor(t) else torch.from_numpy(np.ascontiguousarray(t))).contiguous()
            x = x.pin_memory().to(dev, non_blocking=True)
        return resize(x, scale, out)
