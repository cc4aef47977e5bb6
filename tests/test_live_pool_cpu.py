"""Host logic of the live pool (pgtformer_b200/video.py::LivePool): its schedule against the reference's window loop
for random interleavings of streams, a host model of its ring, the argument checks that run before any device work,
and its device step (Engine.pool_step) on the CPU launch recorder of test_walk_cpu.py, extended to the scatter."""
import random

import numpy as np
import pytest
import torch

from pgtformer_b200.video import LivePool, window_indices
from test_walk_cpu import _engine, _frames as _split, install


class _NoDevice:
    """A model stand-in whose engine must never be reached."""

    def __init__(self):
        self.engine_calls = 0

    def parameters(self):
        yield torch.zeros(1)

    def engine(self):
        self.engine_calls += 1
        raise AssertionError('device work started')


def _tagged(stream, j, hw=(64, 64)):
    """Frame j of stream `stream`, which says so in its first two pixels."""
    f = np.zeros(hw + (3,), np.uint8)
    f[0, 0, 0], f[0, 1, 0] = stream, j
    return f


def _tag(f):
    return int(f[0, 0, 0]), int(f[0, 1, 0])


class _HostRing:
    """A host model of the pool's device step: ring row -> tag of the frame last scattered there.  A window returns
    the tags of the rows it gathers, so a stream reads back the frames its windows name."""

    def __init__(self, pool):
        self.rows, self.steps = {}, []
        pool._step = self.step

    def step(self, hw, new, wins):
        slots = [s for s, _ in new]
        assert len(set(slots)) == len(slots)
        for slot, t in new:
            self.rows[slot] = _tag(t)
        self.steps.append((len(new), len(wins)))
        return [tuple(self.rows[r] for r in win) for win in wins]


def _schedule(seed, lengths, max_streams):
    """A seeded random interleaving: streams open when there is room (staggered starts), each step pushes a random
    non-empty subset of the open streams that still have frames (others stall), and a stream with all its frames
    pushed may be flushed between other streams' pushes."""
    rnd = random.Random(seed)
    waiting, open_, ops = list(range(len(lengths))), {}, []
    pushed = {}
    while waiting or open_:
        if waiting and len(open_) < max_streams and (not open_ or rnd.random() < 0.4):
            k = waiting.pop(0)
            open_[k] = True
            pushed[k] = 0
            ops.append(('open', k))
            continue
        done = [k for k in open_ if pushed[k] == lengths[k]]
        live = [k for k in open_ if pushed[k] < lengths[k]]
        if done and (not live or rnd.random() < 0.3):
            k = rnd.choice(done)
            del open_[k]
            ops.append(('flush', k))
            continue
        if not live:
            continue
        sub = rnd.sample(live, rnd.randint(1, len(live)))
        ops.append(('push', sub))
        for k in sub:
            pushed[k] += 1
    return ops


def _run(pool, ops, frame=_tagged):
    """Plays a schedule on pool; -> {stream: [what each window returned]} in frame order."""
    handles, got, pushed = {}, {}, {}
    for op, arg in ops:
        if op == 'open':
            handles[arg], got[arg], pushed[arg] = pool.open(), [], 0
        elif op == 'flush':
            got[arg].append(pool.flush(handles.pop(arg)))
        else:
            res = pool.push({handles[k]: frame(k, pushed[k]) for k in arg})
            for k in arg:
                assert (res[handles[k]] is None) == (pushed[k] == 0)
                if pushed[k]:
                    got[k].append(res[handles[k]])
                pushed[k] += 1
    return got


@pytest.mark.parametrize('seed', range(12))
def test_random_interleavings_follow_the_reference_window_loop(seed):
    lengths = [1, 2, 3, 5, 7, 11]
    random.Random(seed).shuffle(lengths)
    S = 1 + seed % 5
    pool = LivePool(_NoDevice(), S)
    host = _HostRing(pool)
    got = _run(pool, _schedule(seed, lengths, S))
    for k, n in enumerate(lengths):
        assert got[k] == [tuple((k, j) for j in win) for win in window_indices(n)], (k, n)
    assert all(B <= S and Bw <= S and B + Bw > 0 for B, Bw in host.steps)


def test_streams_never_share_ring_rows():
    """Every stream's new frames go to its own three rows while it is open; a freed stream's rows are reused."""
    pool = LivePool(_NoDevice(), 3)
    seen = []
    pool._step = lambda hw, new, wins: seen.append([s for s, _ in new]) or [None] * len(wins)
    a, b, c = pool.open(), pool.open(), pool.open()
    for j in range(4):
        pool.push({a: _tagged(0, j), b: _tagged(1, j), c: _tagged(2, j)})
    assert [sorted(s // 3 for s in step) for step in seen] == [[0, 1, 2]] * 4
    assert [[s % 3 for s in step] for step in seen] == [[j % 3] * 3 for j in range(4)]
    pool.flush(b)
    d = pool.open()
    pool.push({d: _tagged(3, 0), a: _tagged(0, 4)})
    assert seen[-1] == [3 * 1 + 0, 3 * 0 + 4 % 3]                # d takes b's rows, a keeps its own


def test_open_past_max_streams_raises():
    pool = LivePool(_NoDevice(), 2)
    h = pool.open()
    pool.open()
    with pytest.raises(ValueError):
        pool.open()
    pool.close(h)
    pool.open()
    with pytest.raises(ValueError):
        LivePool(_NoDevice(), 0)


def _bad_pushes(pool, a, b):
    ok = np.zeros((64, 64, 3), np.uint8)
    return [
        {a: np.zeros((64, 64, 3), np.float32)},                      # dtype
        {a: torch.zeros(64, 64, 3, dtype=torch.int32)},
        {a: np.zeros((1, 64, 64, 3), np.uint8)},                     # rank
        {a: np.zeros((64, 64), np.uint8)},
        {a: np.zeros((64, 64, 4), np.uint8)},                        # not rgb24
        {a: np.zeros((96, 64, 3), np.uint8)},                        # not multiples of 64
        {a: ok, b: np.zeros((64, 100, 3), np.uint8)},
        {a: ok, b: np.zeros((128, 64, 3), np.uint8)},                # two sizes in one step
        {a: ok, 12345: ok},                                          # unknown handle
        {a: ok, 'x': ok},
        [(a, ok), (b, ok), (a, ok)],                                 # a handle listed twice
    ]


@pytest.mark.parametrize('case', range(11))
def test_bad_arguments_raise_before_any_device_work(case):
    model = _NoDevice()
    pool = LivePool(model, 2)
    a, b = pool.open(), pool.open()
    with pytest.raises(ValueError):
        pool.push(_bad_pushes(pool, a, b)[case])
    assert model.engine_calls == 0
    assert pool._streams == {a: [0, 0], b: [1, 0]}               # nothing was counted


def test_closed_handles_and_size_changes_raise_before_any_device_work():
    model = _NoDevice()
    pool = LivePool(model, 2)
    host = _HostRing(pool)
    a, b = pool.open(), pool.open()
    pool.push({a: _tagged(0, 0)})
    for bad in ({b: np.zeros((64, 128, 3), np.uint8)},               # the pool holds 64 x 64 frames
                {a: np.zeros((128, 64, 3), np.uint8)}):
        with pytest.raises(ValueError, match='changed'):
            pool.push(bad)
    pool.flush(a)
    for call in (lambda: pool.push({a: _tagged(0, 1)}), lambda: pool.flush(a), lambda: pool.close(a)):
        with pytest.raises(ValueError, match='unknown or closed'):
            call()
    assert model.engine_calls == 0 and len(host.steps) == 2
    assert pool.flush(b) is None                                     # a stream without frames restores nothing
    c = pool.open()
    assert pool.push({c: _tagged(2, 0, (128, 64))}) == {c: None}     # an empty pool takes a new size
    assert pool.push({}) == {}


@pytest.fixture
def recorder(monkeypatch):
    return install(monkeypatch)


def _recorded_pool(eng, S, H, W, w, rec, drop_stats=False):
    """A LivePool whose steps run Engine.pool_step on the CPU recorder, on host buffers laid out as _PoolState's."""
    from pgtformer_b200 import ops
    pool = LivePool(_NoDevice(), S, w=w)
    ring = eng.live_ring(H, W, w, S)
    u8 = torch.zeros(4 * S, H, W, 3, dtype=torch.uint8)
    x = torch.empty(S, 3, H, W)
    out = torch.empty(S, H, W, 3, dtype=torch.uint8)
    scatter = ops.scatter_frames

    def maybe_drop(x, idx, out):
        if drop_stats and out is ring.get('h_stats'):
            return out
        return scatter(x, idx, out)

    def step(hw, new, wins):
        slots = torch.tensor([s for s, _ in new], dtype=torch.int32) if new else None
        index = torch.tensor([r for win in wins for r in win], dtype=torch.int32) if wins else None
        for k, (_, t) in enumerate(new):
            u8[3 * S + k] = torch.as_tensor(t)
        ops.scatter_frames = maybe_drop
        try:
            eng.pool_step(u8, x, ring, slots, index, w, True, out[:len(wins)])
        finally:
            ops.scatter_frames = scatter
        return list(wins)
    pool._step = step
    return pool, ring


def _install_scatter(monkeypatch, rec):
    """The recorder of test_walk_cpu.py, plus the two calls only the pool step makes: the rgb24 conversion (a fresh
    write) and the scatter, which moves each frame's content — and the statistics it holds — to its slot."""
    from pgtformer_b200 import ops

    def u8hwc_to_f32nchw(x_u8, out):
        rec.log.append(('u8hwc_to_f32nchw', (tuple(x_u8.shape), tuple(out.shape)), False, False))
        for k in _split(out, out.shape[0]):
            rec.held[k] = next(rec.tokens)
        return out

    def scatter_frames(x, idx_i32, out):
        rec.log.append(('scatter_frames', (tuple(x.shape), tuple(idx_i32.shape), tuple(out.shape)), False, False))
        assert x.is_contiguous() and out.is_contiguous() and x.shape[1:] == out.shape[1:]
        src, dst = _split(x, x.shape[0]), _split(out, out.shape[0])
        for i, j in enumerate(idx_i32.tolist()):
            rec.held[dst[j]] = rec.held.get(src[i], ('unknown', next(rec.tokens)))
        return out
    monkeypatch.setattr(ops, 'u8hwc_to_f32nchw', u8hwc_to_f32nchw)
    monkeypatch.setattr(ops, 'scatter_frames', scatter_frames)


@pytest.mark.parametrize('H,W,w', [(64, 64, 1.0), (64, 64, 0.0), (128, 128, 1.0)])
def test_windows_read_the_statistics_of_their_frames_through_scatter_and_gather(network_g, recorder, monkeypatch,
                                                                                H, W, w):
    _install_scatter(monkeypatch, recorder)
    eng = _engine('PGTFormer', network_g)
    pool, ring = _recorded_pool(eng, 3, H, W, w, recorder)
    assert 'h_stats' in ring
    _run(pool, _schedule(7, [5, 2, 4, 3], 3), frame=lambda k, j: _tagged(k, j, (H, W)))
    assert not recorder.violations, '\n'.join(recorder.violations[:10])
    names = [e[0] for e in recorder.log]
    assert 'scatter_frames' in names and 'gather_frames' in names
    assert sum(e[0] == 'groupnorm_apply_stats' and e[3] for e in recorder.log) > 0


def test_the_recorder_sees_statistics_left_behind(network_g, recorder, monkeypatch):
    """The check above has teeth: a step that scatters every entry but h's statistics leaves the windows reading the
    statistics of another frame, and the recorder says so."""
    _install_scatter(monkeypatch, recorder)
    eng = _engine('PGTFormer', network_g)
    pool, _ = _recorded_pool(eng, 2, 64, 64, 1.0, recorder, drop_stats=True)
    _run(pool, _schedule(3, [4, 3], 2))
    assert any('statistics of another tensor' in v for v in recorder.violations)
