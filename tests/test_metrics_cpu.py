"""PSNR / SSIM without a GPU: the numpy restatement of basicsr's calculate_psnr / calculate_ssim
(oracle/metrics_oracle.py) at its closed-form cases and against basicsr's cv2.filter2D form; the host half of the
device scores (metrics.finish), whose PSNR must be bit for bit the oracle's; and the argument checks of metrics.score
and VideoRestorer.evaluate, which must reject bad input before any device work."""
import math

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as MO
from test_live_pool_cpu import _NoDevice


def _pair(hw, seed, kind='random'):
    rs = np.random.RandomState(seed)
    a = rs.randint(0, 256, size=tuple(hw) + (3,), dtype=np.uint8)
    if kind == 'random':
        return a, rs.randint(0, 256, size=a.shape, dtype=np.uint8)
    # smoothed plus noise: a blurred copy of a with small perturbations, the regime restored frames are in
    s = a.astype(np.float64)
    for ax in (0, 1):
        s = (np.roll(s, 1, ax) + 2 * s + np.roll(s, -1, ax)) / 4
    b = np.clip(np.rint(s + rs.normal(0, 4, a.shape)), 0, 255).astype(np.uint8)
    return a, b


def test_identical_frames_score_inf_and_exactly_one():
    from pgtformer_b200 import metrics
    for hw in ((11, 11), (64, 64), (100, 37)):
        a, _ = _pair(hw, hw[1])
        assert MO.psnr(a, a) == float('inf') and MO.sse(a, a) == 0
        assert MO.ssim(a, a) == 1.0 and (MO.ssim_channels(a, a) == 1.0).all()
    got = metrics.finish(np.zeros(2, np.int64), np.ones((2, 3)), (64, 64))
    assert (got['psnr'] == float('inf')).all() and (got['ssim'] == 1.0).all()


@pytest.mark.parametrize('d', [1, 3, 17, 100])
def test_a_uniform_offset_gives_the_closed_form_psnr(d):
    rs = np.random.RandomState(d)
    a = rs.randint(d, 256 - d, size=(48, 40, 3)).astype(np.uint8)
    sign = rs.choice([-1, 1], size=a.shape)
    b = (a.astype(int) + sign * d).astype(np.uint8)
    assert MO.sse(a, b) == d * d * a.size
    assert MO.psnr(a, b) == pytest.approx(10 * math.log10(255.0 ** 2 / d ** 2), rel=1e-15, abs=0)


def test_psnr_from_the_exact_sse_is_the_oracles_bit_for_bit():
    """metrics.finish forms PSNR from an integer sse as basicsr does from the frames: every value equal, not close."""
    from pgtformer_b200 import metrics
    for k, hw in enumerate([(11, 11), (64, 64), (100, 37), (128, 192), (512, 512)]):
        pairs = [_pair(hw, 10 * k + j, 'random' if j % 2 else 'smooth') for j in range(4)]
        got = metrics.finish(np.array([MO.sse(a, b) for a, b in pairs]), np.zeros((4, 3)), hw)['psnr']
        ref = np.array([MO.psnr(a, b) for a, b in pairs])
        assert got.dtype == np.float64 and np.array_equal(got.view(np.int64), ref.view(np.int64)), (hw, got - ref)


@pytest.mark.parametrize('hw', [(512, 512), (64, 64), (128, 192)])
@pytest.mark.parametrize('kind', ['random', 'smooth'])
def test_direct_oracle_equals_basicsr_cv2_form(hw, kind):
    pytest.importorskip('cv2')
    a, b = _pair(hw, hw[0] + hw[1], kind)
    d, c = MO.ssim_channels(a, b), MO.ssim_channels_cv2(a, b)
    assert np.abs(d - c).max() <= 1e-12, np.abs(d - c).max()
    assert abs(MO.ssim(a, b) - MO.ssim(a, b, cv2_form=True)) <= 1e-12


def test_gaussian_window_is_cv2s():
    cv2 = pytest.importorskip('cv2')
    assert np.abs(MO.gaussian_window() - cv2.getGaussianKernel(11, 1.5)[:, 0]).max() <= 1e-16


def test_channel_order_does_not_change_the_scores():
    a, b = _pair((40, 52), 5, 'smooth')
    assert MO.psnr(a[..., ::-1], b[..., ::-1]) == MO.psnr(a, b)
    assert MO.ssim(a[..., ::-1], b[..., ::-1]) == pytest.approx(MO.ssim(a, b), abs=1e-15)


def test_oracle_rejects_frames_below_the_window():
    a = np.zeros((10, 64, 3), np.uint8)
    with pytest.raises(ValueError):
        MO.ssim(a, a)
    with pytest.raises(ValueError):
        MO.psnr(a[:, :, :2], a[:, :, :2])


# ------------------------------------------------------------------ argument checks before any device work
@pytest.fixture
def no_device(monkeypatch):
    from pgtformer_b200 import metrics

    def fail(*a, **k):
        raise AssertionError('device work started')
    monkeypatch.setattr(metrics.ops, 'frame_scores', fail)
    monkeypatch.setattr(metrics, '_on', fail)
    monkeypatch.setattr(torch.Tensor, 'pin_memory', fail)


BAD_PAIRS = [  # (restored, gt)
    (np.zeros((2, 64, 64, 3), np.uint8), np.zeros((2, 64, 48, 3), np.uint8)),          # shapes differ
    (np.zeros((2, 64, 64, 3), np.uint8), np.zeros((3, 64, 64, 3), np.uint8)),          # frame counts differ
    (np.zeros((2, 64, 64, 3), np.float32), np.zeros((2, 64, 64, 3), np.uint8)),        # not uint8
    (np.zeros((2, 64, 64, 3), np.uint8), torch.zeros(2, 64, 64, 3, dtype=torch.int16)),
    (np.zeros((2, 10, 64, 3), np.uint8), np.zeros((2, 10, 64, 3), np.uint8)),          # below 11 x 11
    (torch.zeros(1, 64, 8, 3, dtype=torch.uint8), torch.zeros(1, 64, 8, 3, dtype=torch.uint8)),
    (np.zeros((2, 64, 64), np.uint8), np.zeros((2, 64, 64), np.uint8)),                # not rgb24
    (np.zeros((2, 64, 64, 4), np.uint8), np.zeros((2, 64, 64, 4), np.uint8)),
]


@pytest.mark.parametrize('case', range(len(BAD_PAIRS)))
def test_score_rejects_bad_frames_before_device_work(no_device, case):
    from pgtformer_b200 import metrics
    restored, gt = BAD_PAIRS[case]
    with pytest.raises(ValueError):
        metrics.score(restored, gt)


def test_score_of_no_frames_does_no_device_work(no_device):
    from pgtformer_b200 import metrics
    got = metrics.score(np.zeros((0, 32, 32, 3), np.uint8), torch.zeros(0, 32, 32, 3, dtype=torch.uint8))
    assert got['psnr'].shape == (0,) and got['ssim'].shape == (0,) and got['psnr'].dtype == np.float64


BAD_EVALUATIONS = [  # (frames, gt, size)
    (np.zeros((3, 64, 64, 3), np.uint8), np.zeros((3, 64, 128, 3), np.uint8), None),     # gt not at the frames' size
    (np.zeros((3, 16, 16, 3), np.uint8), np.zeros((3, 16, 16, 3), np.uint8), (64, 64)),  # gt not at `size`
    (np.zeros((3, 16, 16, 3), np.uint8), np.zeros((3, 128, 64, 3), np.uint8), (64, 128)),
    (np.zeros((3, 64, 64, 3), np.uint8), np.zeros((2, 64, 64, 3), np.uint8), None),      # one gt frame short
    (np.zeros((3, 64, 64, 3), np.uint8), np.zeros((3, 64, 64, 3), np.float64), None),    # gt not uint8
    (np.zeros((3, 64, 64, 3), np.uint8), np.zeros((3, 64, 64), np.uint8), None),
    (np.zeros((3, 8, 8, 3), np.uint8), np.zeros((3, 8, 8, 3), np.uint8), None),          # below 11 x 11
    (np.zeros((3, 64, 64, 3), np.int32), np.zeros((3, 64, 64, 3), np.uint8), None),      # frames not uint8
    (np.zeros((3, 16, 16, 3), np.uint8), np.zeros((3, 64, 64, 3), np.uint8), (64, 60)),  # size not multiples of 64
]


@pytest.mark.parametrize('case', range(len(BAD_EVALUATIONS)))
def test_evaluate_rejects_bad_arguments_before_device_work(case):
    from pgtformer_b200.video import VideoRestorer
    frames, gt, size = BAD_EVALUATIONS[case]
    model = _NoDevice()
    with pytest.raises(ValueError):
        VideoRestorer(model).evaluate(frames, gt, size)
    assert model.engine_calls == 0


def test_evaluate_of_no_frames_does_no_device_work():
    from pgtformer_b200.video import VideoRestorer
    model = _NoDevice()
    out, scores = VideoRestorer(model).evaluate(np.zeros((0, 16, 16, 3), np.uint8), np.zeros((0, 64, 128, 3), np.uint8),
                                               size=(64, 128))
    assert out.shape == (0, 64, 128, 3) and scores['psnr'].shape == (0,) and scores['ssim'].shape == (0,)
    assert model.engine_calls == 0
