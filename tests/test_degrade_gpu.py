"""The `lr` degradation on the GPU: pgt_imresize_u8hwc_to_f32nchw bit for bit against the exact-rounding form of
oracle/degrade_oracle.py (step-edge content, so overshoot outside [0, 1] must survive); pgt_f32nchw_resize_to_f32nchw
against the oracle's fma form and, on an AVX2 / AVX512 host, CPU F.interpolate; the ctypes and torch.ops bindings
and argument checks; VideoRestorer.restore / stream / evaluate(downscale=...) byte for byte against the reference's
window loop on the oracle upsampling of degrade.downsample's frames, eager and replayed from CUDA graphs; and the
downscale=None paths, which must launch and write what they did before."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import degrade_oracle as DO
from test_degrade_cpu import bars
from test_live_pool_gpu import _same, model  # noqa: F401  (module fixture)
from test_lr_input_gpu import _bits_equal, _torch_fma_path

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ the imresize kernel
KERNEL_CASES = [  # (frames, source, scale)
    (1, (512, 512), 0.25), (2, (512, 512), 0.25), (48, (64, 64), 0.25), (3, (100, 37), 0.25), (2, (37, 100), 0.25),
    (2, (192, 128), 0.5), (1, (512, 512), 1 / 3), (3, (128, 192), 0.25), (2, (192, 128), 1 / 3), (4, (7, 7), 0.25),
    (1, (720, 480), 0.25), (2, (333, 65), 0.2), (1, (130, 70), 0.125),
]


@pytest.mark.parametrize('n,src,scale', KERNEL_CASES)
def test_imresize_equals_the_exact_oracle(n, src, scale):
    from pgtformer_b200 import degrade
    x = bars(n, src, n + src[0] + src[1])
    got = degrade.downsample(x, scale)
    ref = DO.imresize_exact(x, scale)
    _bits_equal(got, ref)
    if min(src) >= 37:
        assert ref.min() < 0 and ref.max() > 1                 # overshoot reached the output unclamped


def test_downsample_takes_numpy_host_and_cuda_frames():
    from pgtformer_b200 import degrade
    x = bars(3, (100, 64), 5)
    a = degrade.downsample(x)
    assert a.is_cuda and a.dtype == torch.float32 and tuple(a.shape) == (3, 3, 25, 16)
    for t in (torch.from_numpy(x), torch.from_numpy(x).cuda(), torch.from_numpy(x).cuda()[1:]):
        b = degrade.downsample(t)
        assert torch.equal(b.view(torch.int32), a[3 - b.shape[0]:].view(torch.int32))
    assert tuple(degrade.downsample(x[:0]).shape) == (0, 3, 25, 16)


# ------------------------------------------------------------------ the fp32 bilinear resize
RESIZE_CASES = [  # (frames, source, target)
    (2, (128, 128), (512, 512)), (3, (25, 10), (128, 192)), (1, (171, 171), (512, 512)), (4, (16, 16), (64, 64)),
    (2, (1, 1), (64, 64)), (16, (128, 128), (512, 512)), (2, (43, 64), (192, 128)), (1, (512, 512), (512, 512)),
]


def _planes(n, hw, seed):
    """fp32 planes with values outside [0, 1], as imresize leaves them."""
    return np.random.RandomState(seed).uniform(-0.15, 1.15, (n, 3) + tuple(hw)).astype(np.float32)


@pytest.mark.parametrize('n,src,size', RESIZE_CASES)
def test_f32_resize_equals_the_oracle_and_interpolate(n, src, size):
    from pgtformer_b200 import ops
    x = _planes(n, src, n + src[0])
    out = torch.full((n, 3) + size, float('nan'), device='cuda')
    ops.f32nchw_resize_to_f32nchw(torch.from_numpy(x).cuda(), out)
    _bits_equal(out, DO.upsample_f32(x, size))
    if _torch_fma_path(size):
        _bits_equal(out, F.interpolate(torch.from_numpy(x), size, mode='bilinear', align_corners=True).numpy())


def test_u8_resize_keeps_its_bits_after_the_loader_template():
    """The rgb24 instantiation of the shared resize kernel against the fp32 one on the same unit values."""
    from pgtformer_b200 import ops
    x = np.random.RandomState(2).randint(0, 256, (3, 37, 53, 3)).astype(np.uint8)
    a = ops.u8hwc_resize_to_f32nchw(torch.from_numpy(x).cuda(), torch.empty(3, 3, 128, 192, device='cuda'), (37, 53))
    b = ops.f32nchw_resize_to_f32nchw(torch.from_numpy(DO.unit(x)).cuda(), torch.empty(3, 3, 128, 192, device='cuda'))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------ bindings and argument checks
def test_ctypes_and_torch_ops_give_the_same_bits():
    from pgtformer_b200 import degrade, ops, torch_ops
    pgt = torch_ops.load()
    x = torch.from_numpy(bars(3, (100, 37), 9)).cuda()
    a = degrade.downsample(x)
    th, tw = degrade.plan((100, 37), 0.25)
    b = torch.empty_like(a)
    pgt.imresize_u8hwc_to_f32nchw(x, th[0].cuda(), th[1].cuda(), tw[0].cuda(), tw[1].cuda(), b)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    c = ops.f32nchw_resize_to_f32nchw(a, torch.empty(3, 3, 128, 64, device='cuda'))
    d = torch.empty_like(c)
    pgt.f32nchw_resize_to_f32nchw(a, d)
    assert torch.equal(c.view(torch.int32), d.view(torch.int32))


def test_bad_arguments_are_rejected():
    from pgtformer_b200 import _lib, degrade, ops
    lib = _lib.load()
    x = torch.zeros(1, 64, 64, 3, dtype=torch.uint8, device='cuda')
    (wh, ih, _, _), _ = degrade.plan((64, 64), 0.25)
    wh, ih = wh.cuda(), ih.cuda()
    y = torch.empty(2 * 3 * 64 * 64 + 1, device='cuda')
    for args in ((x.data_ptr(), 1, 64, 64, wh.data_ptr(), ih.data_ptr(), 0, 16, wh.data_ptr(), ih.data_ptr(), 16, 16),
                 (x.data_ptr(), 1, 64, 64, wh.data_ptr(), ih.data_ptr(), 16, 65, wh.data_ptr(), ih.data_ptr(), 16, 16),
                 (x.data_ptr(), 0, 64, 64, wh.data_ptr(), ih.data_ptr(), 16, 16, wh.data_ptr(), ih.data_ptr(), 16, 16),
                 (x.data_ptr(), 1, 64, 64, None, ih.data_ptr(), 16, 16, wh.data_ptr(), ih.data_ptr(), 16, 16)):
        assert lib.pgt_imresize_u8hwc_to_f32nchw(*args, y.data_ptr(), None) != 0
    f = torch.zeros(1, 3, 16, 16, device='cuda')
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.f32nchw_resize_to_f32nchw(f, torch.empty(1, 3, 96, 64, device='cuda'))          # H % 64
    assert lib.pgt_f32nchw_resize_to_f32nchw(f.data_ptr(), 1, 16, 16, 64, 64, y.data_ptr() + 4, None) != 0
    assert lib.pgt_f32nchw_resize_to_f32nchw(f.data_ptr(), 1, 0, 16, 64, 64, y.data_ptr(), None) != 0


# ------------------------------------------------------------------ VideoRestorer against the reference's loop
VIDEO_CASES = [  # (n, ground truth, scale, size)
    (5, (64, 64), 0.25, None),
    (4, (128, 192), 0.25, None),
    (3, (192, 128), 1 / 3, None),
    (3, (100, 37), 0.25, (64, 64)),
]


_ORACLE = {}


def _oracle(model, n, src, scale, size):
    """The case's ground truth and the reference's window loop on its `lr` input (computed once per module)."""
    key = (n, src, scale, size)
    if key not in _ORACLE:
        from pgtformer_b200 import degrade
        frames = bars(n, src, n + src[1])

        def window(x):
            with torch.no_grad():
                return model(torch.from_numpy(x).cuda(), w=1.0, adain=True)[0][1].float().cpu().numpy()
        lowres = lambda win: degrade.downsample(win, scale).cpu().numpy()     # noqa: E731
        _ORACLE[key] = frames, np.stack(DO.restore_frames(list(frames), window, lowres, size or src))
    return _ORACLE[key]


@pytest.mark.parametrize('clips', [1, 2, 5])
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('n,src,scale,size', VIDEO_CASES)
def test_video_restorer_equals_the_oracle_loop(model, n, src, scale, size, graph, clips):
    from pgtformer_b200.video import VideoRestorer
    frames, ref = _oracle(model, n, src, scale, size)
    got = VideoRestorer(model, clips_per_batch=clips, cuda_graph=graph).restore(frames, size, downscale=scale)
    _same(got, ref)


def test_stream_equals_restore_with_downscale(model):
    from pgtformer_b200.video import VideoRestorer
    frames = bars(7, (128, 192), 4)
    vr = VideoRestorer(model, clips_per_batch=3)
    _same(np.stack(list(vr.stream(iter(frames), downscale=0.25))), vr.restore(frames, downscale=0.25))
    _same(np.stack(list(vr.stream(iter(frames), size=(64, 64), downscale=1 / 3))),
          vr.restore(frames, (64, 64), downscale=1 / 3))


@pytest.mark.parametrize('graph', [False, True])
def test_evaluate_is_the_lr_protocol(model, graph):
    from pgtformer_b200 import metrics
    from pgtformer_b200.video import VideoRestorer
    gt = bars(5, (128, 192), 6)
    vr = VideoRestorer(model, clips_per_batch=2, cuda_graph=graph)
    restored, scores = vr.evaluate(gt, gt, downscale=0.25)
    _same(restored, VideoRestorer(model, clips_per_batch=2).restore(gt, downscale=0.25))
    ref = metrics.score(restored, gt)
    for k in ('psnr', 'ssim'):
        assert np.array_equal(scores[k].view(np.int64), ref[k].view(np.int64)), k


@pytest.mark.parametrize('graph', [False, True])
def test_downscale_none_launches_and_writes_what_it_did(model, graph):
    from pgtformer_b200 import ops
    from pgtformer_b200.video import VideoRestorer
    frames = bars(4, (64, 64), 8)
    vr = VideoRestorer(model, clips_per_batch=2, cuda_graph=graph)
    a = vr.restore(frames)                                          # warms up (and captures) both paths' shapes
    vr.restore(frames, downscale=None)
    counts = []
    for kw in ({}, {'downscale': None}):
        ops.reset_launch_count()
        got = vr.restore(frames, **kw)
        torch.cuda.synchronize()
        counts.append(ops.launch_count())
        _same(got, a)
    assert counts[0] == counts[1]
