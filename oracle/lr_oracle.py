"""TEST INFRASTRUCTURE — numpy restatement of the low-resolution input of the reference's test set, used only by tests/
as the checker for the device upsampling (pgt_u8hwc_resize_to_f32nchw) and the `size=` path of pgtformer_b200/video.py.
Not a product path.

Restates `data/vfhq_full_dataset.py:1046-1051` (the `LR_Blind` frames of `VFHQFULLntmeBASICV2TESTUP`, `is_aligned:
false`, no mean / std):

    lq = np.array(np.array(frames) / 255.0, np.float32)                    # [t,h,w,c]
    lq = torch.from_numpy(lq).permute(0, 3, 1, 2)
    lq = F.interpolate(lq, (512, 512), mode='bilinear', align_corners=True)

with F.interpolate spelled out as torch's CPU kernel evaluates it on an AVX2 / AVX512 host: per axis, in fp32,
scale = (in - 1) / (out - 1) (0 for out = 1), src = scale * o, i0 = min(floor(src), in - 1), i1 = i0 + (i0 < in - 1),
l1 = clamp(src - i0, 0, 1), l0 = 1 - l1; then out = fma(h0, fma(w0, a, w1 b), h1 fma(w0, c, w1 d)) with every product
rounded to fp32 and every fma rounded once.  The fma is emulated exactly (fma32): an fp32 product is exact in float64,
the float64 sum is made round-to-odd from its exact error term, and round-to-odd at 53 bits followed by one rounding to
24 bits is the correctly rounded fp32 result.

`restore_frames` is the reference's window loop (`inference.py:12-76`, oracle/video_oracle.py) with this transform in
place of `rgbnp2tensor`.
"""
import numpy as np

from . import video_oracle as VO


def fma32(a, b, c):
    """fp32 fma(a, b, c), rounded once (numpy arrays or scalars, broadcast)."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b                                            # exact: 24 + 24 bits fit in 53
    s = p + c
    bp = s - c                                           # TwoSum: p + c == s + e exactly
    e = (p - bp) + (c - (s - bp))
    even = (s.view(np.int64) & 1) == 0
    toward = np.where(e > 0, np.inf, -np.inf)
    s = np.where((e != 0) & even, np.nextafter(s, toward), s)     # round to odd
    return s.astype(np.float32)


def lerp_axis(n_in, n_out):
    """(i0, i1, l0, l1) of every output position along one axis, as torch computes them (align_corners=True)."""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    src = np.float32(scale) * np.arange(n_out, dtype=np.float32)
    i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    return i0, i1, l0, l1


def upsample(frames_u8, size):
    """rgb24 frames [t,h,w,3] uint8 -> float32 [t,3,H,W]: data/vfhq_full_dataset.py:1046-1051 at size = (H, W)."""
    H, W = size
    frames = np.asarray(frames_u8)
    unit = np.moveaxis(np.array(np.array(frames) / 255.0, np.float32), 3, 1)        # [t,3,h,w]
    h, w = unit.shape[2:]
    y0, y1, h0, h1 = lerp_axis(h, H)
    x0, x1, w0, w1 = lerp_axis(w, W)
    r0, r1 = unit[:, :, y0, :], unit[:, :, y1, :]
    a, b, c, d = r0[..., x0], r0[..., x1], r1[..., x0], r1[..., x1]
    h0, h1 = h0[:, None], h1[:, None]
    top = fma32(w0, a, w1 * b)
    bot = fma32(w0, c, w1 * d)
    return np.ascontiguousarray(fma32(h0, top, h1 * bot))


def restore_frames(frames, model_window, size):
    """inference.py:12-76 over source frames of any size, restored at size = (H, W): each window's three frames go
    through `upsample` (in place of rgbnp2tensor) and model_window(float32 [3,3,H,W]) -> the restored middle frame
    float32 [3,H,W], kept as clamp(x, 0, 1) * 255 truncated to uint8."""
    return VO.restore_frames(frames, lambda win: VO.tensor2rgb(model_window(upsample(np.stack(win), size))))
