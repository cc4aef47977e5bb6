"""Host logic of per-stream settings in a live pool (pgtformer_b200/video.py::LivePool.open / configure and
LiveRestorer.configure): defaults and overrides, the argument checks that run before any device work, how a step's
windows split into a batch without the SFT fusion and one with it, the per-frame weights and AdaIN flags a step
uploads, the graph keys, and when the ring is rebuilt to keep the SFT skip tensors.  The device step runs on a stub
engine that records what the pool asks of it."""
import contextlib

import pytest
import torch

from pgtformer_b200 import ops
from pgtformer_b200.video import LivePool, LiveRestorer
from test_live_pool_cpu import _NoDevice, _tagged


class _StubEngine:
    """Records the pool's device calls.  Each restored window writes the ring row of its middle frame into pixel
    (0, 0, 0) of its output, so a test can tell which window each returned frame came from."""

    def __init__(self):
        self.dev = torch.device('cpu')
        self.rings, self.calls, self.captures = [], [], []

    def live_ring(self, H, W, w, streams=1):
        ring = {'feats': {2: torch.zeros(4 * streams)} if w > 0 else {}}
        self.rings.append(w > 0)
        return ring

    def frame_step(self, x, slot, ring):
        self.calls.append(('frame_step', slot))

    def _restore(self, kind, index, w, adain, out_u8):
        rows = index.tolist()
        wt = w.tolist() if torch.is_tensor(w) else w
        self.calls.append((kind, rows, wt, adain.tolist()))
        for i in range(len(rows) // 3):
            out_u8[i, 0, 0, 0] = rows[3 * i + 1]

    def pool_step(self, u8, x, ring, slots, index, w, adain, out_u8):
        if slots is not None:
            self.calls.append(('frames', slots.tolist()))
        if index is not None:
            assert not torch.is_tensor(w) and w == 0.0
            self._restore('plain', index, w, adain, out_u8)

    def window_step(self, index, w, adain, ring, out_u8):
        assert torch.is_tensor(w) and w.dtype == torch.float32 and (w > 0).all()
        assert ring['feats'], 'fused windows on a ring without the skip tensors'
        self._restore('fused', index, w, adain, out_u8)

    def _capture(self, run, pool=None):
        key = self.captures.append(None) or len(self.captures) - 1
        eng = self

        class Graph:
            def replay(self):
                eng.calls.append(('replay', key))
                run()

            def pool(self):
                return 'pool'
        return Graph(), None


class _Model:
    def __init__(self):
        self.eng = _StubEngine()

    def parameters(self):
        yield torch.zeros(1)

    def engine(self):
        return self.eng


class _Event:
    def record(self, *a):
        pass

    def synchronize(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    """A model on the stub engine, with the CUDA calls of _PoolState made host no-ops."""
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(ops, 'u8hwc_to_f32nchw', lambda x_u8, out: out)     # the recompute's rgb24 conversion
    return _Model()


def _steps(eng, kind):
    return [c for c in eng.calls if c[0] == kind]


# ------------------------------------------------------------------ settings and argument checks
def test_streams_take_the_pool_defaults_or_their_own():
    pool = LivePool(_NoDevice(), 4, w=0.5, adain=False)
    a, b, c = pool.open(), pool.open(w=1.0), pool.open(adain=True)
    d = pool.open(w=0.0, adain=True)
    conf = {h: pool._conf[pool._streams[h][0]] for h in (a, b, c, d)}
    assert conf == {a: (0.5, False), b: (1.0, False), c: (0.5, True), d: (0.0, True)}
    pool.configure(a, w=0.3)
    pool.configure(b, adain=True)
    pool.configure(c)
    assert pool._conf[pool._streams[a][0]] == (0.3, False)
    assert pool._conf[pool._streams[b][0]] == (1.0, True)
    assert pool._conf[pool._streams[c][0]] == (0.5, True)
    pool.close(a)
    e = pool.open()                                              # a's rows, the pool's defaults
    assert pool._streams[e][0] == 0 and pool._conf[0] == (0.5, False)


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf'), 'nan'])
def test_non_finite_w_raises_before_any_device_work(bad):
    model = _NoDevice()
    with pytest.raises(ValueError):
        LivePool(model, 2, w=bad)
    with pytest.raises(ValueError):
        LiveRestorer(model, w=bad)
    pool = LivePool(model, 2)
    with pytest.raises(ValueError):
        pool.open(w=bad)
    assert pool._streams == {}                                   # no handle was taken
    h = pool.open(w=0.7)
    with pytest.raises(ValueError):
        pool.configure(h, w=bad)
    assert pool._conf[0] == (0.7, True)
    live = LiveRestorer(model, w=0.25)
    with pytest.raises(ValueError):
        live.configure(w=bad)
    assert (live.w, live.adain) == (0.25, True)
    assert model.engine_calls == 0


def test_configure_on_closed_or_unknown_handles_raises():
    pool = LivePool(_NoDevice(), 2)
    a = pool.open()
    pool.close(a)
    for h in (a, 12345, 'x', None):
        with pytest.raises(ValueError, match='unknown or closed'):
            pool.configure(h, w=0.5)


# ------------------------------------------------------------------ the step on the stub engine
def _push_all(pool, hs, j, hw=(64, 64)):
    return pool.push({h: _tagged(k, j, hw) for k, h in enumerate(hs)})


@pytest.mark.parametrize('graph', [False, True])
def test_windows_split_by_w_and_upload_their_settings(stub, graph):
    """w <= 0 windows (a negative w included) go to the batch without fusion, the others to the fused batch with one
    weight per frame; every frame carries its stream's AdaIN flag; each stream gets its own window back."""
    settings = [(1.0, True), (0.0, False), (0.3, False), (-2.0, True), (0.5, True)]
    pool = LivePool(stub, 5, cuda_graph=graph)
    hs = [pool.open(w=w, adain=a) for w, a in settings]
    _push_all(pool, hs, 0)
    got = _push_all(pool, hs, 1)
    eng = stub.eng
    plain, fused = _steps(eng, 'plain')[-1], _steps(eng, 'fused')[-1]
    mids = lambda rows: rows[1::3]                               # noqa: E731
    assert mids(plain[1]) == [3 * 1 + 0, 3 * 3 + 0]              # streams 1 and 3: frame 0 of each
    assert plain[3] == [0] * 3 + [1] * 3
    assert mids(fused[1]) == [0, 3 * 2 + 0, 3 * 4 + 0]
    assert fused[2] == pytest.approx([1.0] * 3 + [0.3] * 3 + [0.5] * 3)
    assert fused[3] == [1] * 3 + [0] * 3 + [1] * 3
    assert {h: int(f[0, 0, 0]) for h, f in got.items()} == {h: 3 * k for k, h in enumerate(hs)}


@pytest.mark.parametrize('graph', [False, True])
def test_configure_applies_to_the_next_window(stub, graph):
    pool = LivePool(stub, 2, cuda_graph=graph)
    a, b = pool.open(w=0.0, adain=False), pool.open(w=0.5)
    eng = stub.eng
    _push_all(pool, [a, b], 0)
    _push_all(pool, [a, b], 1)
    assert _steps(eng, 'fused')[-1][2] == pytest.approx([0.5] * 3) and _steps(eng, 'plain')[-1][3] == [0] * 3
    pool.configure(a, w=1.0, adain=True)
    pool.configure(b, w=0.0)
    n = len(eng.calls)
    _push_all(pool, [a, b], 2)
    fused, plain = [c for c in eng.calls[n:] if c[0] == 'fused'], [c for c in eng.calls[n:] if c[0] == 'plain']
    assert fused[-1][1][1::3] == [1] and fused[-1][2] == pytest.approx([1.0] * 3) and fused[-1][3] == [1] * 3
    assert plain[-1][1][1::3] == [3 + 1] and plain[-1][3] == [1] * 3
    pool.configure(a, w=0.25)
    n = len(eng.calls)
    pool.flush(a)                                                # the flushed frame takes the new setting
    assert [c[2] for c in eng.calls[n:] if c[0] == 'fused'] == [pytest.approx([0.25] * 3)]


def test_live_restorer_configure_reaches_its_stream_and_the_next(stub):
    live = LiveRestorer(stub, w=0.0, adain=False, cuda_graph=False)
    eng = stub.eng
    live.push(_tagged(0, 0))
    live.push(_tagged(0, 1))
    assert _steps(eng, 'plain')[-1][3] == [0] * 3 and not _steps(eng, 'fused')
    live.configure(w=0.75)
    live.push(_tagged(0, 2))
    assert _steps(eng, 'fused')[-1][2] == pytest.approx([0.75] * 3) and _steps(eng, 'fused')[-1][3] == [0] * 3
    live.configure(adain=True)
    live.flush()
    assert _steps(eng, 'fused')[-1][3] == [1] * 3
    live.push(_tagged(1, 0))                                     # a new stream keeps the settings
    live.push(_tagged(1, 1))
    assert _steps(eng, 'fused')[-1][2] == pytest.approx([0.75] * 3) and _steps(eng, 'fused')[-1][3] == [1] * 3


def test_graph_keys_count_new_frames_windows_and_windows_without_fusion(stub):
    pool = LivePool(stub, 3)
    a, b, c = pool.open(w=1.0), pool.open(w=0.0), pool.open(w=0.5, adain=False)
    _push_all(pool, [a, b, c], 0)
    for j in (1, 2, 3):
        _push_all(pool, [a, b, c], j)
    pool.push({a: _tagged(0, 4)})
    pool.push({b: _tagged(1, 4)})
    pool.configure(c, w=0.0)
    pool.push({a: _tagged(0, 5), c: _tagged(2, 4)})
    pool.configure(a, w=-1.0)                                    # b keeps the skip tensors: no rebuild
    pool.configure(b, w=0.3)
    pool.push({a: _tagged(0, 6), c: _tagged(2, 5)})
    pool.flush(b)
    state = pool._state
    assert stub.eng.rings == [True]
    assert list(state.graphs) == [(3, 0), (3, 3, 1), (1, 1), (1, 1, 1), (2, 2, 1), (2, 2, 2), (0, 1)]
    replays = [c[1] for c in stub.eng.calls if c[0] == 'replay']
    assert replays == [0, 1, 1, 1, 2, 3, 4, 5, 6]                # the steady steps replay one graph
    bound = (3 + 1) ** 2 * (3 + 2) // 2 - 1
    assert len(state.graphs) <= bound


def test_the_ring_gains_the_skip_tensors_when_a_stream_reaches_w_above_0(stub):
    """A state built without the skip tensors is rebuilt with them when a stream reaches w > 0 (by open or
    configure), recomputing the frames still inside a window from the rgb24 rows the pool keeps; it keeps them when no
    stream needs them any more."""
    pool = LivePool(stub, 2, w=0.0)
    eng = stub.eng
    a = pool.open()
    pool.push({a: _tagged(0, 0)})
    pool.push({a: _tagged(0, 1)})
    assert eng.rings == [False]
    b = pool.open(w=0.5)                                         # open reaches w > 0
    n = len(eng.calls)
    pool.push({a: _tagged(0, 2), b: _tagged(1, 0)})
    assert eng.rings == [False, True]
    assert [c for c in eng.calls[n:] if c[0] == 'frame_step'][:2] == [('frame_step', 0), ('frame_step', 1)]
    pool.push({a: _tagged(0, 3), b: _tagged(1, 1)})
    assert eng.rings == [False, True]                            # no rebuild while the settings hold
    fused = len(_steps(eng, 'fused'))
    pool.configure(b, w=0.0)
    pool.close(a)
    pool.push({b: _tagged(1, 2)})
    c = pool.open()
    pool.push({b: _tagged(1, 3), c: _tagged(0, 0)})
    pool.push({b: _tagged(1, 4), c: _tagged(0, 1)})
    assert eng.rings == [False, True] and len(_steps(eng, 'fused')) == fused     # kept; no stream fuses
    assert _steps(eng, 'plain')[-1][1][1::3] == [3 + 0, 0]
    pool2 = LivePool(stub, 1, w=0.0)
    d = pool2.open()
    pool2.push({d: _tagged(0, 0)})
    pool2.push({d: _tagged(0, 1)})
    pool2.configure(d, w=1.0)                                    # configure reaches w > 0
    n = len(eng.calls)
    pool2.push({d: _tagged(0, 2)})
    assert eng.rings == [False, True, False, True]
    assert [c for c in eng.calls[n:] if c[0] == 'frame_step'][:2] == [('frame_step', 0), ('frame_step', 1)]
    assert _steps(eng, 'fused')[-1][2] == pytest.approx([1.0] * 3)


def test_uniform_pools_keep_their_ring_and_graph_keys(stub):
    """A pool whose streams share one setting builds one state, keyed as before settings were per stream."""
    for w, keys in ((1.0, [(2, 0), (2, 2), (0, 1)]), (0.0, [(2, 0), (2, 2, 2), (0, 1, 1)])):
        stub.eng.rings.clear()
        pool = LivePool(stub, 2, w=w)
        a, b = pool.open(), pool.open()
        for j in range(3):
            _push_all(pool, [a, b], j)
        pool.flush(a)
        assert stub.eng.rings == [w > 0] and list(pool._state.graphs) == keys
