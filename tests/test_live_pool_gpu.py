"""The live pool (pgtformer_b200/video.py::LivePool) on the GPU: pgt_scatter_frames against index_copy_, every stream
of a pool byte for byte what VideoRestorer.restore gives on that stream alone (itself pinned to the reference loop by
test_video_gpu.py), eager and replayed from CUDA graphs, new weights mid-stream as LiveRestorer takes them, two pools
on one model, and a steady state that replays one graph."""
import numpy as np
import pytest
import torch

from test_live_pool_cpu import _NoDevice, _schedule

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def model(network_g):
    from archs.pgtformer_arch import PGTFormer
    kw = dict(network_g)
    kw.pop('type', None)
    m = PGTFormer(**kw).cuda()
    m.eval()
    m.cuda_graph = False
    return m


# ------------------------------------------------------------------ the kernel
@pytest.mark.parametrize('frame_bytes', [16, 48, 4096 + 16, 512 * 512 * 3, 256 * 256 * 128 * 2])
def test_scatter_frames_equals_index_copy(frame_bytes):
    from pgtformer_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(frame_bytes % 1000)
    for n in range(1, 17):
        rows = 2 * n + 1
        x = torch.randint(0, 256, (n, frame_bytes), dtype=torch.uint8, device='cuda', generator=g)
        y = torch.randint(0, 256, (rows, frame_bytes), dtype=torch.uint8, device='cuda', generator=g)
        idx = torch.randperm(rows, device='cuda', generator=g)[:n].to(torch.int32)
        ref = y.clone().index_copy_(0, idx.long(), x)
        ops.scatter_frames(x, idx, y)
        assert torch.equal(y, ref), n
        if frame_bytes >= 4096:
            break                                                 # the big rows: n = 1 and the wide case below
    if frame_bytes >= 4096:
        n = 16 if frame_bytes < 2 ** 24 else 4
        x = torch.randint(0, 256, (n, frame_bytes), dtype=torch.uint8, device='cuda', generator=g)
        y = torch.zeros(n + 3, frame_bytes, dtype=torch.uint8, device='cuda')
        idx = torch.randperm(n + 3, device='cuda', generator=g)[:n].to(torch.int32)
        assert torch.equal(ops.scatter_frames(x, idx, y), torch.zeros_like(y).index_copy_(0, idx.long(), x))


def test_scatter_frames_rejects_misaligned_and_odd_sizes():
    from pgtformer_b200 import ops
    buf = torch.zeros(4096, dtype=torch.uint8, device='cuda')
    idx = torch.tensor([1, 0], dtype=torch.int32, device='cuda')
    ok = buf[:64].view(2, 32)
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.scatter_frames(buf[8:72].view(2, 32), idx, buf[1024:1088].view(2, 32))      # x misaligned
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.scatter_frames(ok, idx, buf[1032:1096].view(2, 32))                       # y misaligned
    with pytest.raises(RuntimeError, match='libpgt_b200'):
        ops.scatter_frames(buf[:48].view(2, 24), idx, buf[1024:1072].view(2, 24))     # 24-byte frames


# ------------------------------------------------------------------ byte-exact streams
def _video(n, H, W, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(n, H, W, 3), dtype=np.uint8)


def _same(got, ref):
    assert got.shape == ref.shape and got.dtype == np.uint8
    assert np.array_equal(got, ref), 'max |d| = %d' % np.abs(got.astype(int) - ref.astype(int)).max()


def _play(pool, ops, videos, cuda_frames=()):
    """Plays a schedule (test_live_pool_cpu._schedule) with real frames; -> {stream: restored frames}."""
    handles, got, pushed = {}, {}, {}
    for op, arg in ops:
        if op == 'open':
            handles[arg], got[arg], pushed[arg] = pool.open(), [], 0
        elif op == 'flush':
            got[arg].append(pool.flush(handles.pop(arg)))
        else:
            frames = {}
            for k in arg:
                f = videos[k][pushed[k]]
                frames[handles[k]] = torch.from_numpy(f).cuda() if k in cuda_frames else f
            res = pool.push(frames)
            for k in arg:
                assert (res[handles[k]] is None) == (pushed[k] == 0)
                if pushed[k]:
                    got[k].append(res[handles[k]])
                pushed[k] += 1
    return {k: np.stack(v) for k, v in got.items()}


CASES = [  # (H, W, w, adain, lengths, max_streams, seed)
    (64, 64, 1.0, True, [1, 2, 3, 5, 7, 11], 5, 0),
    (64, 64, 0.0, True, [11, 5, 1, 3], 3, 1),
    (64, 64, 1.0, False, [2, 7, 3, 5], 4, 2),
    (64, 64, 0.0, False, [3, 1, 5, 2], 2, 3),
    (128, 192, 1.0, True, [5, 3, 7], 3, 4),
    (128, 192, 0.0, False, [2, 5], 2, 5),
    (512, 512, 1.0, True, [3, 5], 2, 6),
]


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('H,W,w,adain,lengths,S,seed', CASES)
def test_every_stream_equals_video_restorer_alone(model, H, W, w, adain, lengths, S, seed, graph):
    from pgtformer_b200.video import LivePool, VideoRestorer
    videos = [_video(n, H, W, 100 * seed + k) for k, n in enumerate(lengths)]
    pool = LivePool(model, S, w=w, adain=adain, cuda_graph=graph)
    got = _play(pool, _schedule(seed, lengths, S), videos, cuda_frames={1})
    for k, v in enumerate(videos):
        _same(got[k], VideoRestorer(model, w=w, adain=adain, clips_per_batch=4).restore(v))
    if graph:
        assert len(pool._state.graphs) <= (S + 1) ** 2 - 1


def test_cuda_frame_on_another_device_raises_before_any_device_work():
    from pgtformer_b200.video import LivePool
    model = _NoDevice()                                           # parameters on the CPU
    pool = LivePool(model, 1)
    with pytest.raises(ValueError, match='model on cpu'):
        pool.push({pool.open(): torch.zeros(64, 64, 3, dtype=torch.uint8, device='cuda')})
    assert model.engine_calls == 0


@pytest.mark.parametrize('graph', [False, True])
def test_new_weights_mid_stream_match_live_restorer(network_g, graph):
    """load_state_dict() between two steps of a pool: each stream's frames equal what a LiveRestorer gives on that
    stream with the same weight change at the same point of its stream."""
    from archs.pgtformer_arch import PGTFormer
    from pgtformer_b200.video import LivePool, LiveRestorer
    kw = dict(network_g)
    kw.pop('type', None)
    m = PGTFormer(**kw).cuda().eval()
    m.cuda_graph = False
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    sd1 = {k: v * 0.9 if v.is_floating_point() else v for k, v in sd0.items()}
    videos = [_video(6, 64, 64, 90), _video(5, 64, 64, 91)]
    starts = [0, 2]                                               # stream 1 joins at step 2; weights change at step 3

    def run(push, flush):
        """push({stream: frame}) -> {stream: restored or None}; flush(stream) -> its last frame."""
        m.load_state_dict(sd0)
        got = [[], []]
        for step in range(8):
            if step == 3:
                m.load_state_dict(sd1)
            frames = {k: v[step - starts[k]] for k, v in enumerate(videos) if 0 <= step - starts[k] < len(v)}
            for k, r in push(frames).items():
                if r is not None:
                    got[k].append(r)
            for k, v in enumerate(videos):
                if step - starts[k] == len(v):
                    got[k].append(flush(k))
        return [np.stack(g) for g in got]

    lives = [LiveRestorer(m, cuda_graph=graph) for _ in videos]
    ref = run(lambda fs: {k: lives[k].push(f) for k, f in fs.items()}, lambda k: lives[k].flush())
    pool = LivePool(m, 2, cuda_graph=graph)
    handles = {}

    def push(fs):
        for k in fs:
            if k not in handles:
                handles[k] = pool.open()
        res = pool.push({handles[k]: f for k, f in fs.items()})
        return {k: res[handles[k]] for k in fs}
    for k, g in enumerate(run(push, lambda k: pool.flush(handles.pop(k)))):
        _same(g, ref[k])
    m.load_state_dict(sd0)
    from pgtformer_b200.video import VideoRestorer
    old = VideoRestorer(m, clips_per_batch=4).restore(videos[0])
    assert not np.array_equal(old[2:], ref[0][2:])               # the new weights did reach the streams
    _same(ref[0][:2], old[:2])


@pytest.mark.parametrize('graph', [False, True])
def test_two_pools_with_different_w_interleave(model, graph):
    from pgtformer_b200.video import LivePool
    lengths = [4, 6, 3]
    videos = [_video(n, 64, 64, 40 + k) for k, n in enumerate(lengths)]
    pools = LivePool(model, 3, w=1.0, cuda_graph=graph), LivePool(model, 3, w=0.0, adain=False, cuda_graph=graph)
    ops = _schedule(11, lengths, 3)
    handles = [{}, {}]
    got = [{k: [] for k in range(3)}, {k: [] for k in range(3)}]
    pushed = {k: 0 for k in range(3)}
    for op, arg in ops:
        for p, pool in enumerate(pools):
            if op == 'open':
                handles[p][arg] = pool.open()
            elif op == 'flush':
                got[p][arg].append(pool.flush(handles[p].pop(arg)))
            else:
                res = pool.push({handles[p][k]: videos[k][pushed[k]] for k in arg})
                for k in arg:
                    if pushed[k]:
                        got[p][k].append(res[handles[p][k]])
        if op == 'push':
            for k in arg:
                pushed[k] += 1
    from pgtformer_b200.video import VideoRestorer
    for p, (w, adain) in enumerate(((1.0, True), (0.0, False))):
        for k, v in enumerate(videos):
            _same(np.stack(got[p][k]), VideoRestorer(model, w=w, adain=adain, clips_per_batch=4).restore(v))


def test_steady_state_replays_one_graph(model):
    from pgtformer_b200 import ops
    from pgtformer_b200.video import LivePool, VideoRestorer
    S, n = 4, 8
    videos = [_video(n, 64, 64, 60 + k) for k in range(S)]
    pool = LivePool(model, S)
    hs = [pool.open() for _ in range(S)]
    got = [[] for _ in range(S)]
    for j in range(n):
        if j == 3:
            keys = set(pool._state.graphs)
            assert keys == {(S, 0), (S, S)}
            replays = []
            for key, g in pool._state.graphs.items():
                g.replay = (lambda r, key: lambda: replays.append(key) or r())(g.replay, key)
            launches = ops.launch_count()
        res = pool.push({h: videos[k][j] for k, h in enumerate(hs)})
        for k, h in enumerate(hs):
            if res[h] is not None:
                got[k].append(res[h])
    assert ops.launch_count() == launches and set(pool._state.graphs) == keys
    assert replays == [(S, S)] * (n - 3)
    for k, h in enumerate(hs):
        got[k].append(pool.flush(h))
        _same(np.stack(got[k]), VideoRestorer(model, clips_per_batch=4).restore(videos[k]))
