"""TEST INFRASTRUCTURE — restatement of the `lr` degradation of the reference's test set, used only by tests/ and
tools/ as the checker for pgt_imresize_u8hwc_to_f32nchw, pgt_f32nchw_resize_to_f32nchw and the `downscale=` path of
pgtformer_b200/video.py.  Not a product path.

`data/vfhq_full_dataset.py:983-988,1017-1024` builds the low-resolution input from the ground truth itself:

    t = imresize(np.array(v, np.float32) / 255.0, 0.25)                # basicsr.utils.matlab_functions.imresize
    lrimages = torch.from_numpy(np.array(lrimages, np.float32)).permute(0, 3, 1, 2)
    d['lq'] = F.interpolate(lrimages, (512, 512), mode='bilinear', align_corners=True)

Three forms of imresize live here:
  * `imresize_basicsr`: basicsr 1.4's imresize (matlab_functions.py) restated in torch float32, `mv` included: the
    reference form, whose sums run in the host BLAS's order;
  * `imresize_exact`: the same transform with each pass defined as the fp32 value nearest to the exact sum of its fp32
    products (ties to even), in numpy: products are exact in float64, summed as a double-double (TwoSum) and rounded
    once through round-to-odd, as lr_oracle.fma32 does.  `exact_fp32` is the same value from fractions.Fraction, which
    the tests use to check this form;
  * the tap tables both use (`taps`), from basicsr's own torch float32 expressions.
`upsample_f32` is lr_oracle.upsample on fp32 planes (lr_oracle's fma32 and lerp_axis), and `restore_frames` the
reference's window loop on the degraded input.
"""
import math
from fractions import Fraction

import numpy as np
import torch

from . import lr_oracle as LO
from . import video_oracle as VO


# ------------------------------------------------------------------ basicsr/utils/matlab_functions.py (basicsr 1.4)
def cubic(x):
    absx = torch.abs(x)
    absx2 = absx ** 2
    absx3 = absx ** 3
    return (1.5 * absx3 - 2.5 * absx2 + 1) * ((absx <= 1).type_as(absx)) + \
        (-0.5 * absx3 + 2.5 * absx2 - 4 * absx + 2) * (((absx > 1) * (absx <= 2)).type_as(absx))


def calculate_weights_indices(in_length, out_length, scale, kernel='cubic', kernel_width=4, antialiasing=True):
    if (scale < 1) and antialiasing:
        kernel_width = kernel_width / scale
    x = torch.linspace(1, out_length, out_length)
    u = x / scale + 0.5 * (1 - 1 / scale)
    left = torch.floor(u - kernel_width / 2)
    p = math.ceil(kernel_width) + 2
    indices = left.view(out_length, 1).expand(out_length, p) + torch.linspace(0, p - 1, p).view(1, p).expand(
        out_length, p)
    distance_to_center = u.view(out_length, 1).expand(out_length, p) - indices
    if (scale < 1) and antialiasing:
        weights = scale * cubic(distance_to_center * scale)
    else:
        weights = cubic(distance_to_center)
    weights_sum = torch.sum(weights, 1).view(out_length, 1)
    weights = weights / weights_sum.expand(out_length, p)
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
    sym_len_e = indices.max() - in_length
    indices = indices + sym_len_s - 1
    return weights, indices, int(sym_len_s), int(sym_len_e)


def _pad(t, dim, s, e):
    """basicsr's symmetric copy along dim: s flipped leading samples, t, e flipped trailing samples."""
    n = t.size(dim)
    shape = list(t.shape)
    shape[dim] = n + s + e
    aug = torch.FloatTensor(*shape)
    aug.narrow(dim, s, n).copy_(t)
    head = t.narrow(dim, 0, s)
    aug.narrow(dim, 0, s).copy_(head.index_select(dim, torch.arange(head.size(dim) - 1, -1, -1).long()))
    tail = t.narrow(dim, n - e, e)
    aug.narrow(dim, s + n, e).copy_(tail.index_select(dim, torch.arange(tail.size(dim) - 1, -1, -1).long()))
    return aug


def imresize_basicsr(img, scale):
    """basicsr's imresize(img, scale) for a numpy float32 image [h,w,c] (antialiasing, cubic) -> numpy float32
    [ceil(h scale), ceil(w scale), c]: the H pass into out_1, then the W pass, each output a `mv` over its taps."""
    img = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).float()
    in_c, in_h, in_w = img.size()
    out_h, out_w = math.ceil(in_h * scale), math.ceil(in_w * scale)
    weights_h, indices_h, hs, he = calculate_weights_indices(in_h, out_h, scale)
    weights_w, indices_w, ws, we = calculate_weights_indices(in_w, out_w, scale)
    img_aug = _pad(img, 1, hs, he)
    out_1 = torch.FloatTensor(in_c, out_h, in_w)
    kernel_width = weights_h.size(1)
    for i in range(out_h):
        idx = int(indices_h[i][0])
        for j in range(in_c):
            out_1[j, i, :] = img_aug[j, idx:idx + kernel_width, :].transpose(0, 1).mv(weights_h[i])
    out_1_aug = _pad(out_1, 2, ws, we)
    out_2 = torch.FloatTensor(in_c, out_h, out_w)
    kernel_width = weights_w.size(1)
    for i in range(out_w):
        idx = int(indices_w[i][0])
        for j in range(in_c):
            out_2[j, :, i] = out_1_aug[j, :, idx:idx + kernel_width].mv(weights_w[i])
    return out_2.numpy().transpose(1, 2, 0)


def lr_basicsr(frames_u8, scale=0.25):
    """The `lr` branch's llq with the reference form: imresize(np.array(v, np.float32) / 255.0) of each rgb24 frame
    [t,h,w,3] -> float32 [t,3,oh,ow]."""
    return np.stack([imresize_basicsr(np.array(v, np.float32) / 255.0, scale).transpose(2, 0, 1)
                     for v in np.asarray(frames_u8)])


# ------------------------------------------------------------------ the exact-rounding form
def taps(in_len, scale):
    """basicsr's taps for one axis: (weights float32 [out, K], source indices int64 [out, K] with the symmetric padding
    folded into [0, in_len))."""
    out_len = math.ceil(in_len * scale)
    w, idx, s, _ = calculate_weights_indices(in_len, out_len, scale)
    q = idx.long().numpy() - s
    src = np.where(q < 0, -q - 1, np.where(q >= in_len, 2 * in_len - q - 1, q))
    return w.numpy().astype(np.float32), src


def _round_odd_to_f32(hi, lo):
    """fp32 nearest to hi + lo (exact float64 pair), ties to even: TwoSum, round to odd at 53 bits, round to 24."""
    s = hi + lo
    bp = s - hi
    t = (hi - (s - bp)) + (lo - bp)
    even = (s.view(np.int64) & 1) == 0
    toward = np.where(t > 0, np.inf, -np.inf)
    s = np.where((t != 0) & even, np.nextafter(s, toward), s)
    return s.astype(np.float32)


def exact_pass(x, w, idx, axis):
    """One pass along `axis` of float32 x: out[..., i, ...] = fp32 nearest to sum_k w[i, k] x[..., idx[i, k], ...]."""
    x = np.moveaxis(np.asarray(x, np.float32), axis, -1).astype(np.float64)
    hi = np.zeros(x.shape[:-1] + (w.shape[0],))
    lo = np.zeros_like(hi)
    for k in range(w.shape[1]):
        p = w[:, k].astype(np.float64) * x[..., idx[:, k]]
        s = hi + p
        bp = s - hi
        lo = lo + ((hi - (s - bp)) + (p - bp))
        hi = s
    return np.moveaxis(_round_odd_to_f32(hi, lo), -1, axis)


def unit(frames_u8):
    """(float)(v / 255.0) of rgb24 frames [t,h,w,3] -> float32 [t,3,h,w]."""
    return np.ascontiguousarray(np.moveaxis(np.array(np.asarray(frames_u8) / 255.0, np.float32), 3, 1))


def imresize_exact(frames_u8, scale=0.25):
    """rgb24 frames [t,h,w,3] -> float32 [t,3,ceil(h scale),ceil(w scale)]: H pass, then W pass on its fp32 result,
    each output the fp32 value nearest to its exact sum."""
    x = unit(frames_u8)
    wh, ih = taps(x.shape[2], scale)
    ww, iw = taps(x.shape[3], scale)
    return np.ascontiguousarray(exact_pass(exact_pass(x, wh, ih, 2), ww, iw, 3))


def exact_fp32(weights, values):
    """The fp32 value nearest to sum(w * x) computed in fractions.Fraction (ties to even)."""
    s = sum((Fraction(float(w)) * Fraction(float(x)) for w, x in zip(weights, values)), Fraction(0))
    f = np.float32(float(s))
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - s), int(np.array(c).view(np.int32)) & 1))
    return np.float32(best)


# ------------------------------------------------------------------ bilinear upsampling of fp32 frames
def upsample_f32(x, size):
    """float32 frames [t,3,h,w] -> float32 [t,3,H,W]: F.interpolate(mode='bilinear', align_corners=True) in the fma
    form torch's AVX2 / AVX512 kernel evaluates (lr_oracle.upsample on fp32 planes)."""
    x = np.asarray(x, np.float32)
    H, W = size
    h, w = x.shape[2:]
    y0, y1, h0, h1 = LO.lerp_axis(h, H)
    x0, x1, w0, w1 = LO.lerp_axis(w, W)
    r0, r1 = x[:, :, y0, :], x[:, :, y1, :]
    a, b, c, d = r0[..., x0], r0[..., x1], r1[..., x0], r1[..., x1]
    h0, h1 = h0[:, None], h1[:, None]
    top = LO.fma32(w0, a, w1 * b)
    bot = LO.fma32(w0, c, w1 * d)
    return np.ascontiguousarray(LO.fma32(h0, top, h1 * bot))


def restore_frames(frames, model_window, lowres, size):
    """inference.py:12-76 on the `lr` protocol: each window's three frames go through lowres (rgb24 [3,h,w,3] ->
    float32 [3,3,oh,ow], the degradation) and upsample_f32 to size, then model_window(float32 [3,3,H,W]) -> the
    restored middle frame float32 [3,H,W], kept as clamp(x, 0, 1) * 255 truncated to uint8."""
    return VO.restore_frames(frames, lambda win: VO.tensor2rgb(model_window(upsample_f32(lowres(np.stack(win)),
                                                                                         size))))
