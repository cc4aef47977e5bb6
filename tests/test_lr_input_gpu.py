"""Low-resolution input on the GPU: pgt_u8hwc_resize_to_f32nchw bit for bit against the numpy restatement of the
reference test set's upsampling (oracle/lr_oracle.py) and, on an AVX2 / AVX512 host, against CPU F.interpolate, for
one size per launch and ragged sizes from the device table; the equal-size case against pgt_u8hwc_to_f32nchw; the
ctypes and torch.ops bindings; VideoRestorer.restore(size=...) byte for byte against the reference's window loop on
the oracle input; and LiveRestorer / LivePool(size=...) streams byte for byte against VideoRestorer.restore(size=...)
on each stream alone, through stalls, flushes, a settings change and new weights."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lr_oracle as LO
from test_live_pool_cpu import _schedule
from test_live_pool_gpu import _play, _same, model  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
AVX = torch.backends.cpu.get_cpu_capability() != 'DEFAULT'


def _torch_fma_path(size):
    """Whether CPU F.interpolate evaluates the fma form the reference's dataloader hosts use at this output size: an
    AVX2 / AVX512 host does, except for a 64 x 64 output, which torch 2.11 computes along another path (DESIGN §6b)."""
    return AVX and tuple(size) != (64, 64)


def _src(n, hw, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(n,) + tuple(hw) + (3,), dtype=np.uint8)


def _bits_equal(got, ref):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert got.shape == ref.shape
    same = got.view(np.int32) == ref.view(np.int32)
    assert same.all(), '%d of %d values differ' % ((~same).sum(), same.size)


def _interpolate(x, size):
    lq = torch.from_numpy(np.array(np.array(x) / 255.0, np.float32)).permute(0, 3, 1, 2)
    return F.interpolate(lq, size, mode='bilinear', align_corners=True).numpy()


# ------------------------------------------------------------------ the kernel
KERNEL_CASES = [  # (frames, source, target)
    (1, (128, 128), (512, 512)), (4, (128, 128), (512, 512)), (48, (16, 16), (64, 64)), (5, (96, 160), (512, 512)),
    (3, (128, 128), (448, 576)), (2, (37, 53), (128, 192)), (3, (1, 1), (64, 64)), (2, (100, 37), (192, 128)),
    (1, (720, 480), (512, 512)), (2, (128, 512), (512, 512)), (7, (3, 200), (64, 128)),
]


@pytest.mark.parametrize('n,src,size', KERNEL_CASES)
def test_kernel_equals_the_oracle_and_interpolate(n, src, size):
    from pgtformer_b200 import ops
    x = _src(n, src, n * 1000 + src[0])
    out = torch.full((n, 3) + size, float('nan'), device='cuda')
    ops.u8hwc_resize_to_f32nchw(torch.from_numpy(x).cuda(), out, src)
    ref = LO.upsample(x, size)
    _bits_equal(out, ref)
    if _torch_fma_path(size):
        _bits_equal(out, _interpolate(x, size))


@pytest.mark.parametrize('size', [(64, 64), (128, 192), (512, 512)])
def test_ragged_sizes_from_the_device_table_at_any_offset(size):
    """One launch over frames of different sizes, each at its own byte offset (the pool's staging rows, and a table
    whose offsets skip and reorder bytes), from a base that is not aligned."""
    from pgtformer_b200 import ops
    H, W = size
    srcs = [(1, 1), (16, 16), (H // 4, W // 4), (37, 53), (H, W), (H // 2, W), (5, 3 * W)]
    frames = [_src(1, s, 7 * k + H)[0] for k, s in enumerate(srcs)]
    for rows in (True, False):
        base = 3
        if rows:
            offs = [k * H * W * 3 for k in range(len(srcs))]
        else:
            offs, o = [], len(srcs) * 11
            for f in reversed(frames):
                offs.insert(0, o)
                o += f.size + 5
        buf = np.random.RandomState(H).randint(0, 256, base + max(offs) + H * W * 3 * 2, dtype=np.uint8)
        for f, o in zip(frames, offs):
            buf[base + o:base + o + f.size] = f.reshape(-1)
        dbuf = torch.from_numpy(buf).cuda()
        table = torch.tensor([[h, w, o] for (h, w), o in zip(srcs, offs)], dtype=torch.int32, device='cuda')
        out = torch.full((len(srcs), 3, H, W), float('nan'), device='cuda')
        ops.u8hwc_resize_to_f32nchw(dbuf[base:], out, (H, W), table)
        for k, f in enumerate(frames):
            _bits_equal(out[k:k + 1], LO.upsample(f[None], size))
            if _torch_fma_path(size):
                _bits_equal(out[k:k + 1], _interpolate(f[None], size))


@pytest.mark.parametrize('n,size', [(1, (64, 64)), (5, (128, 192)), (16, (512, 512))])
def test_equal_sizes_equal_the_plain_conversion(n, size):
    from pgtformer_b200 import ops
    x = torch.from_numpy(_src(n, size, n)).cuda()
    a = ops.u8hwc_to_f32nchw(x, torch.empty((n, 3) + size, device='cuda'))
    b = ops.u8hwc_resize_to_f32nchw(x, torch.empty((n, 3) + size, device='cuda'), size)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_ctypes_and_torch_op_give_the_same_bits():
    from pgtformer_b200 import ops, torch_ops
    pgt = torch_ops.load()
    x = torch.from_numpy(_src(3, (37, 53), 1)).cuda()
    a = ops.u8hwc_resize_to_f32nchw(x, torch.empty(3, 3, 128, 192, device='cuda'), (37, 53))
    b = torch.empty_like(a)
    pgt.u8hwc_resize_to_f32nchw(x, 37, 53, None, b)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    table = torch.tensor([[37, 53, 0], [20, 10, 100], [37, 53, 37 * 53 * 3 * 2]], dtype=torch.int32, device='cuda')
    c, d = torch.empty_like(a), torch.empty_like(a)
    ops.u8hwc_resize_to_f32nchw(x, c, (37, 53), table)
    pgt.u8hwc_resize_to_f32nchw(x, 37, 53, table, d)
    assert torch.equal(c.view(torch.int32), d.view(torch.int32)) and torch.equal(c[2], a[2])


def test_bad_arguments_are_rejected():
    from pgtformer_b200 import _lib, ops
    x = torch.zeros(64, 64, 3, dtype=torch.uint8, device='cuda')
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.u8hwc_resize_to_f32nchw(x, torch.empty(1, 3, 96, 64, device='cuda'), (16, 16))     # H % 64
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.u8hwc_resize_to_f32nchw(x, torch.empty(1, 3, 64, 64, device='cuda'), (0, 16))
    lib = _lib.load()
    y = torch.empty(2 * 3 * 64 * 64 + 1, device='cuda')
    rc = lib.pgt_u8hwc_resize_to_f32nchw(x.data_ptr(), 1, 8, 8, None, 64, 64, y.data_ptr() + 4, None)   # misaligned y
    assert rc != 0


# ------------------------------------------------------------------ VideoRestorer against the reference's loop
def _oracle_loop(model, frames, size, w, adain):
    """inference.py:12-76 with the test set's upsampling: each window's oracle input through PGTFormer.forward."""
    def window(x):
        with torch.no_grad():
            return model(torch.from_numpy(x).cuda(), w=w, adain=adain)[0][1].float().cpu().numpy()
    return np.stack(LO.restore_frames(list(frames), window, size))


VIDEO_CASES = [  # (n, source, size, w, adain)
    (5, (16, 16), (64, 64), 1.0, True),
    (4, (16, 16), (64, 64), 0.0, False),
    (6, (32, 48), (128, 192), 0.5, False),
    (3, (32, 48), (128, 192), 1.0, True),
    (5, (37, 53), (128, 192), 0.0, True),
    (4, (37, 53), (128, 192), 0.5, True),
    (3, (128, 128), (512, 512), 1.0, True),
    (2, (128, 128), (512, 512), 0.0, False),
]


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('n,src,size,w,adain', VIDEO_CASES)
def test_video_restorer_equals_the_oracle_loop(model, n, src, size, w, adain, graph):
    from pgtformer_b200.video import VideoRestorer
    frames = _src(n, src, n + src[1] + int(10 * w))
    got = VideoRestorer(model, w=w, adain=adain, clips_per_batch=2, cuda_graph=graph).restore(frames, size)
    _same(got, _oracle_loop(model, frames, size, w, adain))


def test_stream_equals_restore_with_size(model):
    from pgtformer_b200.video import VideoRestorer
    frames = _src(7, (37, 53), 3)
    vr = VideoRestorer(model, clips_per_batch=3)
    _same(np.stack(list(vr.stream(iter(frames), size=(128, 192)))), vr.restore(frames, size=(128, 192)))


@pytest.mark.parametrize('graph', [False, True])
def test_sources_at_the_model_size_equal_the_default_path(model, graph):
    from pgtformer_b200.video import LivePool, VideoRestorer
    frames = _src(5, (128, 192), 8)
    ref = VideoRestorer(model, clips_per_batch=2, cuda_graph=graph).restore(frames)
    _same(VideoRestorer(model, clips_per_batch=2, cuda_graph=graph).restore(frames, size=(128, 192)), ref)
    pool = LivePool(model, 2, cuda_graph=graph, size=(128, 192))
    got = _play(pool, [('open', 0), ('push', [0]), ('push', [0]), ('push', [0]), ('push', [0]), ('push', [0]),
                       ('flush', 0)], [frames])
    _same(got[0], ref)


# ------------------------------------------------------------------ live streams against VideoRestorer
POOL_CASES = [  # (size, [(frames, source) per stream], max_streams, w, adain, seed)
    ((64, 64), [(5, (16, 16)), (3, (64, 64)), (1, (16, 16)), (7, (8, 40)), (4, (33, 17)), (2, (1, 1))], 4, 1.0, True,
     0),
    ((64, 64), [(6, (16, 16)), (4, (20, 12))], 2, 0.0, False, 1),
    ((128, 192), [(4, (32, 48)), (5, (37, 53)), (3, (128, 192))], 3, 0.5, True, 2),
    ((512, 512), [(3, (128, 128)), (4, (96, 160))], 2, 1.0, True, 3),
]


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('size,streams,S,w,adain,seed', POOL_CASES)
def test_pool_streams_equal_video_restorer_alone(model, size, streams, S, w, adain, seed, graph):
    from pgtformer_b200.video import LivePool, VideoRestorer
    videos = [_src(n, hw, 50 * seed + k) for k, (n, hw) in enumerate(streams)]
    pool = LivePool(model, S, w=w, adain=adain, cuda_graph=graph, size=size)
    got = _play(pool, _schedule(seed, [n for n, _ in streams], S), videos, cuda_frames={1})
    for k, v in enumerate(videos):
        _same(got[k], VideoRestorer(model, w=w, adain=adain, clips_per_batch=4).restore(v, size))
    if graph:
        assert len(pool._state.graphs) <= (S + 1) ** 2 - 1


@pytest.mark.parametrize('graph', [False, True])
def test_live_restorer_equals_video_restorer(model, graph):
    from pgtformer_b200.video import LiveRestorer, VideoRestorer
    live = LiveRestorer(model, w=0.5, cuda_graph=graph, size=(128, 192))
    for n, hw, seed in ((5, (37, 53), 1), (1, (16, 16), 2), (3, (128, 192), 3)):       # streams of three sizes
        v = _src(n, hw, seed)
        _same(np.stack(list(live.stream(v))), VideoRestorer(model, w=0.5, clips_per_batch=4).restore(v, (128, 192)))


@pytest.mark.parametrize('graph', [False, True])
def test_settings_change_and_new_weights_mid_stream(network_g, graph):
    """Two streams of different source sizes; stream 0 changes w and AdaIN at step 2 (its frames from 1 on), the
    weights change at step 4.  Each stream equals a LiveRestorer(size=...) with the same changes at the same points,
    and before the weight change VideoRestorer.restore(size=...)."""
    from archs.pgtformer_arch import PGTFormer
    from pgtformer_b200.video import LivePool, LiveRestorer, VideoRestorer
    kw = dict(network_g)
    kw.pop('type', None)
    m = PGTFormer(**kw).cuda().eval()
    m.cuda_graph = False
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    sd1 = {k: v * 0.9 if v.is_floating_point() else v for k, v in sd0.items()}
    size = (64, 64)
    videos = [_src(7, (16, 16), 70), _src(6, (24, 40), 71)]
    starts = [0, 1]

    def run(push, flush, configure):
        m.load_state_dict(sd0)
        got = [[], []]
        for step in range(9):
            if step == 2:
                configure(0, 0.0, False)
            if step == 4:
                m.load_state_dict(sd1)
            frames = {k: v[step - starts[k]] for k, v in enumerate(videos) if 0 <= step - starts[k] < len(v)}
            for k, r in push(frames).items():
                if r is not None:
                    got[k].append(r)
            for k, v in enumerate(videos):
                if step - starts[k] == len(v):
                    got[k].append(flush(k))
        return [np.stack(g) for g in got]

    lives = [LiveRestorer(m, cuda_graph=graph, size=size) for _ in videos]
    ref = run(lambda fs: {k: lives[k].push(f) for k, f in fs.items()}, lambda k: lives[k].flush(),
              lambda k, w, a: lives[k].configure(w=w, adain=a))
    pool = LivePool(m, 2, cuda_graph=graph, size=size)
    handles = {}

    def push(fs):
        for k in fs:
            if k not in handles:
                handles[k] = pool.open()
        res = pool.push({handles[k]: f for k, f in fs.items()})
        return {k: res[handles[k]] for k in fs}
    got = run(push, lambda k: pool.flush(handles.pop(k)), lambda k, w, a: pool.configure(handles[k], w=w, adain=a))
    for g, r in zip(got, ref):
        _same(g, r)
    m.load_state_dict(sd0)
    first = VideoRestorer(m, clips_per_batch=4).restore(videos[1], size)
    _same(ref[1][:2], first[:2])                                 # stream 1 before the weight change
    assert not np.array_equal(ref[1][3:], first[3:])             # the new weights did reach it
    zero = VideoRestorer(m, w=0.0, adain=False, clips_per_batch=4).restore(videos[0], size)
    _same(ref[0][1:3], zero[1:3])                                # stream 0 after its settings change
