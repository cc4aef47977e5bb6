"""PSNR / SSIM on the GPU: pgt_frame_scores against the numpy restatement of basicsr's calculate_psnr / calculate_ssim
(oracle/metrics_oracle.py) at frame sizes no tile divides, on random, smoothed-plus-noise, identical and extreme
pairs; its determinism, eager and replayed from a CUDA graph; the ctypes and torch.ops bindings; metrics.score on
host and device inputs; and VideoRestorer.evaluate, whose frames must be restore()'s bytes and whose scores must be
the oracle's on them.  sse is exact and PSNR bit for bit; each channel's SSIM within 1e-12."""
import functools

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as MO
from test_live_pool_gpu import _same, model  # noqa: F401  (module fixture)
from test_metrics_cpu import _pair

pytestmark = pytest.mark.gpu
SIZES = [(512, 512), (128, 192), (64, 64), (11, 11), (100, 37)]
KINDS = ['random', 'smooth', 'identical', 'extremes']
TOL = 1e-12


@functools.lru_cache(maxsize=None)
def _frames(hw, kind, n=17):
    """n frame pairs of one kind and the oracle's sse, PSNR and channel SSIM of each (computed once per module)."""
    a, b = [], []
    for f in range(n):
        if kind == 'extremes':                                 # all 0 against all 255, alternating sides
            x = np.full(tuple(hw) + (3,), 0 if f % 2 else 255, np.uint8)
            y = 255 - x
        else:
            x, y = _pair(hw, 1000 * f + hw[0] + 7 * hw[1], 'random' if kind == 'random' else 'smooth')
            y = x.copy() if kind == 'identical' else y
        a.append(x)
        b.append(y)
    a, b = np.stack(a), np.stack(b)
    ref = (np.array([MO.sse(x, y) for x, y in zip(a, b)]), np.array([MO.psnr(x, y) for x, y in zip(a, b)]),
           np.stack([MO.ssim_channels(x, y) for x, y in zip(a, b)]), np.array([MO.ssim(x, y) for x, y in zip(a, b)]))
    return a, b, ref


def _check(sse, ssim_c, hw, ref, n):
    from pgtformer_b200 import metrics
    r_sse, r_psnr, r_ssim_c, r_ssim = (r[:n] for r in ref)
    sse = sse.cpu().numpy() if torch.is_tensor(sse) else sse
    ssim_c = ssim_c.cpu().numpy() if torch.is_tensor(ssim_c) else ssim_c
    assert np.array_equal(sse, r_sse), (sse, r_sse)
    got = metrics.finish(sse, ssim_c, hw)
    assert np.array_equal(got['psnr'].view(np.int64), r_psnr.view(np.int64)), (got['psnr'], r_psnr)
    err = np.abs(ssim_c - r_ssim_c).max()
    assert err <= TOL, err
    assert np.abs(got['ssim'] - r_ssim).max() <= TOL


# ------------------------------------------------------------------ the kernel
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('hw', SIZES)
@pytest.mark.parametrize('F', [1, 3, 16, 17])
def test_kernel_equals_the_oracle(F, hw, kind):
    from pgtformer_b200 import ops
    a, b, ref = _frames(hw, kind)
    sse, ssim = ops.frame_scores(torch.from_numpy(a[:F]).cuda(), torch.from_numpy(b[:F]).cuda())
    _check(sse, ssim, hw, ref, F)
    if kind == 'identical':
        assert (ssim.cpu() == 1.0).all()


@pytest.mark.parametrize('F,hw', [(16, (512, 512)), (3, (100, 37)), (17, (128, 192))])
def test_runs_and_graph_replays_give_the_same_bits(F, hw):
    from pgtformer_b200 import ops
    a, b, ref = _frames(hw, 'smooth')
    da, db = torch.from_numpy(a[:F]).cuda(), torch.from_numpy(b[:F]).cuda()
    first = ops.frame_scores(da, db)
    for _ in range(3):
        again = ops.frame_scores(da, db)
        assert all(torch.equal(x, y) for x, y in zip(first, again))
    sa, sb = torch.zeros_like(da), torch.zeros_like(db)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.frame_scores(sa, sb)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = ops.frame_scores(sa, sb)
    for src_a, src_b in ((db, da), (da, db)):                   # replays on new inputs, then on the first ones
        sa.copy_(src_a)
        sb.copy_(src_b)
        g.replay()
        eager = ops.frame_scores(src_a, src_b)
        assert all(torch.equal(x, y) for x, y in zip(outs, eager))
    _check(outs[0], outs[1], hw, ref, F)


def test_ctypes_and_torch_op_give_the_same_bits():
    from pgtformer_b200 import ops, torch_ops
    pgt = torch_ops.load()
    a, b, _ = _frames((100, 37), 'random')
    da, db = torch.from_numpy(a[:5]).cuda(), torch.from_numpy(b[:5]).cuda()
    sse, ssim = ops.frame_scores(da, db)
    s2, q2 = torch.empty_like(sse), torch.empty_like(ssim)
    pgt.frame_scores(da, db, s2, q2)
    assert torch.equal(sse, s2) and torch.equal(ssim, q2)


def test_bad_arguments_are_rejected():
    from pgtformer_b200 import _lib, ops
    x = torch.zeros(2, 10, 64, 3, dtype=torch.uint8, device='cuda')
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.frame_scores(x, x)                                              # H < 11
    lib = _lib.load()
    y = torch.zeros(2, 64, 64, 3, dtype=torch.uint8, device='cuda')
    ws = torch.empty(int(lib.pgt_frame_scores_ws_doubles(2, 64, 64)), dtype=torch.float64, device='cuda')
    sse = torch.empty(2, dtype=torch.int64, device='cuda')
    ssim = torch.empty(2, 3, dtype=torch.float64, device='cuda')
    args = [y.data_ptr(), y.data_ptr(), 2, 64, 64, ws.data_ptr(), sse.data_ptr(), ssim.data_ptr(), None]
    assert lib.pgt_frame_scores(*args) == 0
    for k in (0, 1, 5, 6, 7):                                               # each pointer null in turn
        assert lib.pgt_frame_scores(*(args[:k] + [None] + args[k + 1:])) == -1
    assert lib.pgt_frame_scores(*(args[:2] + [0] + args[3:])) == -1        # F = 0
    assert lib.pgt_frame_scores(*(args[:4] + [10] + args[5:])) == -1       # W < 11


# ------------------------------------------------------------------ metrics.score
def test_score_takes_numpy_host_and_device_frames():
    from pgtformer_b200 import metrics
    a, b, ref = _frames((128, 192), 'smooth')
    a, b = a[:5], b[:5]
    for x, y in ((a, b), (torch.from_numpy(a), b), (torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()),
                 (torch.from_numpy(a).cuda(), b), (a, torch.from_numpy(b).cuda())):
        got = metrics.score(x, y)
        assert np.array_equal(got['psnr'].view(np.int64), ref[1][:5].view(np.int64))
        assert np.abs(got['ssim'] - ref[3][:5]).max() <= TOL


# ------------------------------------------------------------------ VideoRestorer.evaluate
EVAL_CASES = [  # (n, source, size)
    (5, (64, 64), None),
    (4, (128, 192), None),
    (5, (64, 64), (128, 128)),
]


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('n,src,size', EVAL_CASES)
def test_evaluate_restores_as_restore_and_scores_as_the_oracle(model, n, src, size, graph):
    from pgtformer_b200.video import VideoRestorer
    rs = np.random.RandomState(n + src[1])
    frames = rs.randint(0, 256, size=(n,) + src + (3,), dtype=np.uint8)
    gt = rs.randint(0, 256, size=(n,) + (size or src) + (3,), dtype=np.uint8)
    vr = VideoRestorer(model, clips_per_batch=2, cuda_graph=graph)
    restored, scores = vr.evaluate(frames, gt, size)
    _same(restored, vr.restore(frames, size))
    ref_psnr = np.array([MO.psnr(x, y) for x, y in zip(restored, gt)])
    assert np.array_equal(scores['psnr'].view(np.int64), ref_psnr.view(np.int64))
    ref_ssim = np.array([MO.ssim(x, y) for x, y in zip(restored, gt)])
    assert np.abs(scores['ssim'] - ref_ssim).max() <= TOL
    self_scores = vr.evaluate(frames, restored, size)[1]                   # scored against itself: inf and 1
    assert (self_scores['psnr'] == float('inf')).all() and (self_scores['ssim'] == 1.0).all()
    if graph:
        eager = VideoRestorer(model, clips_per_batch=2).evaluate(frames, gt, size)
        _same(restored, eager[0])
        for k in ('psnr', 'ssim'):
            assert np.array_equal(scores[k].view(np.int64), eager[1][k].view(np.int64))
