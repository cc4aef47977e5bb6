"""The `lr` degradation on the host: the library's imresize tap tables (pgtformer_b200/degrade.py) against a closed-form
float64 computation of basicsr's taps, the folded padding and the footprint bound the device kernel sizes its shared
memory by; the exact-rounding form of oracle/degrade_oracle.py against fractions.Fraction and against basicsr's own
torch float32 form; and the argument checks, which must all fire before any device work."""
import math

import numpy as np
import pytest
import torch

from oracle import degrade_oracle as DO

# |exact - basicsr| over the cases below; basicsr's fp32 `mv` errs by up to about K 2^-24 sum |w x| per pass.  The
# observed maximum is 2^-22 (2 ulp of 1.0, 4 ulp of values in [0.5, 1)); values near 0 have smaller ulps, so the
# bound is absolute.
BASICSR_BOUND = 2.0 ** -20
CASES = [((512, 512), 0.25), ((100, 37), 0.25), ((192, 128), 0.5), ((512, 512), 1 / 3)]


def bars(n, hw, seed):
    """Random rgb24 frames crossed by 0 / 255 bars, so that bicubic overshoot leaves [0, 1] on both sides."""
    x = np.random.RandomState(seed).randint(0, 256, (n,) + tuple(hw) + (3,)).astype(np.uint8)
    yy, xx = np.meshgrid(np.arange(hw[0]), np.arange(hw[1]), indexing='ij')
    on = (yy // 13) % 3 != 0
    x[:, on & ((xx // 9) % 2 == 0)] = 255
    x[:, on & ((xx // 9) % 2 == 1)] = 0
    x[:, (yy // 11) % 4 == 1, :] = 255 - x[:, (yy // 11) % 4 == 1, :]
    return x


def _closed_form(in_len, scale):
    """basicsr's taps in float64 throughout, trimmed and mirrored the same way, rounded to fp32 at the end."""
    out_len = math.ceil(in_len * scale)
    kw = 4 / scale
    x = np.arange(1, out_len + 1, dtype=np.float64)
    u = x / scale + 0.5 * (1 - 1 / scale)
    left = np.floor(u - kw / 2)
    p = math.ceil(kw) + 2
    idx = left[:, None] + np.arange(p)[None, :]
    a = np.abs((u[:, None] - idx) * scale)
    cub = np.where(a <= 1, 1.5 * a ** 3 - 2.5 * a ** 2 + 1, np.where(a <= 2, -0.5 * a ** 3 + 2.5 * a ** 2 - 4 * a + 2, 0))
    w = scale * cub
    w = w / w.sum(1, keepdims=True)
    zeros = (w == 0).sum(0)
    lo, hi = (1 if zeros[0] else 0), (p - 1 if zeros[-1] else p)
    w, idx = w[:, lo:hi], idx[:, lo:hi].astype(np.int64)
    q = idx - 1
    src = np.where(q < 0, -q - 1, np.where(q >= in_len, 2 * in_len - q - 1, q))
    return w.astype(np.float32), src


@pytest.mark.parametrize('scale', [0.25, 0.5, 1 / 3])
@pytest.mark.parametrize('in_len', [512, 100, 37, 192, 128, 720, 64, 17])
def test_tap_tables_equal_the_closed_form(in_len, scale):
    from pgtformer_b200 import degrade
    if scale == 0.25 and in_len < 7:
        pytest.skip('too small for basicsr')
    w, idx, _, _ = degrade.taps(in_len, scale)
    w, idx = w.numpy(), idx.numpy()
    rw, ridx = _closed_form(in_len, scale)
    assert np.array_equal(idx, ridx) and idx.min() >= 0 and idx.max() < in_len
    assert idx.dtype == np.int32 and w.dtype == np.float32
    if scale in (0.25, 0.5):
        assert np.array_equal(w.view(np.int32), rw.view(np.int32))
    else:
        # basicsr evaluates the cubic's outer piece, -0.5 a^3 + 2.5 a^2 - 4 a + 2, in fp32, and at a = 5/3 its terms
        # cancel: the weights move from the float64 value by up to 50 ulp, at most 6.5e-8 (measured).
        d = np.abs(w.view(np.int32).astype(np.int64) - rw.view(np.int32))
        assert d.max() <= 64 and np.abs(w.astype(np.float64) - rw).max() <= 1e-7
    ow, oi = DO.taps(in_len, scale)                          # the oracle's own restatement: basicsr's bits
    assert np.array_equal(w.view(np.int32), ow.view(np.int32)) and np.array_equal(idx, oi)


def test_quarter_scale_taps_are_dyadic_and_sum_to_one():
    from pgtformer_b200 import degrade
    w, idx, q, a = degrade.taps(512, 0.25)
    assert w.shape == (128, 16) and a == 1.171875 and q == -12
    w64 = w.double()
    assert (w64.sum(1) == 1).all() and float(w.min()) == -75 / 4096
    assert (torch.from_numpy(np.diff(idx.numpy()[2:-2], axis=0)) == 4).all()
    assert int(idx[0, 0]) == 5 and int(idx[-1, -1]) == 506       # 6 samples mirrored at each end
    w, _, _, _ = degrade.taps(37, 0.25)
    assert w.shape == (10, 16)


@pytest.mark.parametrize('scale', [0.25, 0.5, 1 / 3, 0.2, 0.125, 0.75])
@pytest.mark.parametrize('in_len', [7, 37, 100, 512, 721])
def test_tile_footprints_fit_the_kernels_bound(in_len, scale):
    """pgt_imresize_u8hwc_to_f32nchw stages min(n, ceil((T - 1) K / 4) + K + 2) samples per axis for T outputs."""
    from pgtformer_b200 import degrade
    try:
        _, idx, _, _ = degrade.taps(in_len, scale)
    except ValueError:
        return
    idx = idx.numpy()
    K = idx.shape[1]
    for T in (1, 2, 4, 8, 16, 32):
        cap = min(in_len, ((T - 1) * K + 3) // 4 + K + 2)
        for o in range(0, idx.shape[0]):
            rows = idx[o:o + T]
            assert rows.max() - rows.min() + 1 <= cap, (T, o)


@pytest.mark.parametrize('n', range(1, 13))
def test_padding_check_matches_where_basicsr_runs(n):
    from pgtformer_b200 import degrade
    img = np.zeros((n, 16, 3), np.float32)
    try:
        DO.imresize_basicsr(img, 0.25)
        runs = True
    except RuntimeError:
        runs = False
    try:
        degrade.plan((n, 16), 0.25)
        accepted = True
    except ValueError:
        accepted = False
    assert runs == accepted


# ------------------------------------------------------------------ the exact form
def test_exact_form_equals_fractions():
    rs = np.random.RandomState(0)
    for (h, w), s in [((100, 37), 0.25), ((60, 45), 1 / 3)]:
        u = DO.unit(bars(1, (h, w), 3))
        wh, ih = DO.taps(h, s)
        ww, iw = DO.taps(w, s)
        o1 = DO.exact_pass(u, wh, ih, 2)
        o2 = DO.exact_pass(o1, ww, iw, 3)
        for _ in range(150):
            c, i, j, jj = rs.randint(3), rs.randint(o1.shape[2]), rs.randint(w), rs.randint(o2.shape[3])
            assert DO.exact_fp32(wh[i], u[0, c, ih[i], j]).view(np.int32) == o1[0, c, i, j].view(np.int32)
            assert DO.exact_fp32(ww[jj], o1[0, c, i, iw[jj]]).view(np.int32) == o2[0, c, i, jj].view(np.int32)


@pytest.mark.parametrize('hw,scale', CASES)
def test_exact_form_is_within_basicsr_rounding(hw, scale):
    x = bars(2, hw, hw[1])
    e = DO.imresize_exact(x, scale)
    b = DO.lr_basicsr(x, scale)
    assert e.shape == b.shape == (2, 3, math.ceil(hw[0] * scale), math.ceil(hw[1] * scale)) and e.dtype == np.float32
    assert np.abs(e.astype(np.float64) - b).max() <= BASICSR_BOUND
    assert e.min() < 0 and e.max() > 1                       # overshoot is kept


def test_upsample_f32_equals_the_rgb24_form_on_unit_values():
    from oracle import lr_oracle as LO
    x = np.random.RandomState(1).randint(0, 256, (2, 37, 53, 3)).astype(np.uint8)
    a = DO.upsample_f32(DO.unit(x), (128, 192))
    assert np.array_equal(a.view(np.int32), LO.upsample(x, (128, 192)).view(np.int32))


# ------------------------------------------------------------------ argument checks, before any device work
@pytest.mark.parametrize('scale', [0, 1, 1.5, -0.25, float('nan'), 'quarter', None, 0.6])
def test_bad_scales_raise_value_error(scale):
    from pgtformer_b200 import degrade
    with pytest.raises(ValueError):
        degrade.downsample(np.zeros((1, 64, 64, 3), np.uint8), scale)


@pytest.mark.parametrize('frames', [np.zeros((1, 64, 64, 3), np.float32), np.zeros((64, 64, 3), np.uint8),
                                    np.zeros((1, 64, 64, 4), np.uint8), np.zeros((1, 6, 64, 3), np.uint8),
                                    np.zeros((1, 64, 0, 3), np.uint8)])
def test_bad_frames_raise_value_error(frames):
    from pgtformer_b200 import degrade
    with pytest.raises(ValueError):
        degrade.downsample(frames, 0.25)


def test_video_restorer_checks_downscale_first():
    from pgtformer_b200.video import VideoRestorer
    vr = VideoRestorer(None)
    frames = np.zeros((3, 64, 64, 3), np.uint8)
    for kw in (dict(downscale=0), dict(downscale=1.0), dict(downscale='x'), dict(downscale=0.6)):
        with pytest.raises(ValueError):
            vr.restore(frames, **kw)
        with pytest.raises(ValueError):
            vr.evaluate(frames, frames, **kw)
    with pytest.raises(ValueError, match='multiples of 64'):
        vr.restore(np.zeros((3, 100, 64, 3), np.uint8), downscale=0.25)         # the output is the frames' size
    with pytest.raises(ValueError, match='symmetric padding'):
        vr.restore(np.zeros((3, 6, 6, 3), np.uint8), size=(64, 64), downscale=0.25)
    with pytest.raises(ValueError, match='gt_u8'):
        vr.evaluate(frames, np.zeros((3, 128, 128, 3), np.uint8), downscale=0.25)
    with pytest.raises(ValueError):
        vr.stream(iter(frames), downscale=2)
    with pytest.raises(ValueError, match='multiples of 64'):
        next(vr.stream(iter(np.zeros((3, 100, 64, 3), np.uint8)), downscale=0.25))
