"""Low-resolution input on the host: the numpy restatement of the reference test set's upsampling
(oracle/lr_oracle.py) bit for bit against F.interpolate, the `size` and source-frame checks of VideoRestorer,
LiveRestorer and LivePool that run before any device work, and a pool's schedule of source frames on a stub engine:
per-stream source sizes, the size table each step uploads, the staged rows, the capacity rule, the "changed" rule per
stream, the recompute after a rebuild, and graph keys that do not depend on source sizes."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lr_oracle as LO
from pgtformer_b200 import ops
from pgtformer_b200.video import LivePool, LiveRestorer, VideoRestorer
from test_live_pool_cpu import _NoDevice
from test_live_settings_cpu import _Model, _StubEngine, _steps, stub  # noqa: F401  (fixture)

SHAPES = [((128, 128), (512, 512)), ((96, 160), (512, 512)), ((128, 128), (448, 576)), ((64, 64), (512, 512)),
          ((128, 512), (512, 512)), ((720, 480), (512, 512)), ((1, 1), (64, 64)), ((100, 37), (192, 128)),
          ((512, 512), (512, 512))]
RANDOM_SHAPES = [((int(h), int(w)), (64 * int(a), 64 * int(b)))
                 for h, w, a, b in np.random.RandomState(5).randint(1, 9, (4, 4)) * [31, 23, 1, 1]]


# ------------------------------------------------------------------ the oracle transform
@pytest.mark.skipif(torch.backends.cpu.get_cpu_capability() == 'DEFAULT',
                    reason="torch's DEFAULT kernel evaluates bilinear without fma; the reference's x86 hosts use fma")
@pytest.mark.parametrize('src,size', SHAPES + RANDOM_SHAPES)
def test_oracle_equals_interpolate_bit_for_bit(src, size):
    t = 1 if src[0] * src[1] > 100000 else 3
    x = np.random.RandomState(src[0] + size[1]).randint(0, 256, (t,) + src + (3,), dtype=np.uint8)
    lq = torch.from_numpy(np.array(np.array(x) / 255.0, np.float32)).permute(0, 3, 1, 2)
    ref = F.interpolate(lq, size, mode='bilinear', align_corners=True).numpy()
    got = LO.upsample(x, size)
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert np.array_equal(got.view(np.int32), ref.view(np.int32)), float((got != ref).mean())


def test_fma32_rounds_once():
    """(1 - 2^-23) 2^-24 (1 + 2^-23) + (1 + 2^-23) = 1 + 3 2^-24 - 2^-70: the float64 sum rounds to the fp32 tie
    1 + 3 2^-24, which then rounds to even (1 + 2^-22); one rounding of the exact value gives 1 + 2^-23."""
    a, b, c = np.float32(1 - 2 ** -23), np.float32(2 ** -24 * (1 + 2 ** -23)), np.float32(1 + 2 ** -23)
    assert float(np.float32(np.float64(a) * np.float64(b) + np.float64(c))) == 1 + 2 ** -22
    assert float(LO.fma32(a, b, c)) == 1 + 2 ** -23
    assert float(LO.fma32(-a, b, -c)) == -(1 + 2 ** -23)


# ------------------------------------------------------------------ checks before any device work
@pytest.mark.parametrize('bad', [(100, 64), (64, 0), (0, 64), (-64, 64), (64,), (64, 64, 64), 'xy', 64])
def test_size_must_be_multiples_of_64_at_construction(bad):
    model = _NoDevice()
    frames = np.zeros((2, 16, 16, 3), np.uint8)
    for make in (lambda: VideoRestorer(model).restore(frames, size=bad),
                 lambda: VideoRestorer(model).stream(iter(frames), size=bad),
                 lambda: LivePool(model, 2, size=bad), lambda: LiveRestorer(model, size=bad)):
        with pytest.raises(ValueError, match='size'):
            make()
    assert model.engine_calls == 0


def test_size_is_kept_as_ints():
    model = _NoDevice()
    assert LivePool(model, 2, size=(np.int64(128), 64)).size == (128, 64)
    assert LiveRestorer(model, size=(64, 64)).size == (64, 64)
    assert LivePool(model, 2).size is None


def test_source_frames_are_checked_before_any_device_work():
    model = _NoDevice()
    pool = LivePool(model, 2, size=(64, 64))
    a, b = pool.open(), pool.open()
    ok = np.zeros((16, 16, 3), np.uint8)
    bad = [np.zeros((65, 64, 3), np.uint8),                      # more pixels than the model size
           np.zeros((1, 4097, 3), np.uint8),
           np.zeros((0, 16, 3), np.uint8), np.zeros((16, 0, 3), np.uint8),
           np.zeros((16, 16, 3), np.float32), np.zeros((16, 16), np.uint8), np.zeros((16, 16, 4), np.uint8)]
    for f in bad:
        with pytest.raises(ValueError):
            pool.push({a: ok, b: f})
        with pytest.raises(ValueError):
            LiveRestorer(model, size=(64, 64)).push(f)
    assert model.engine_calls == 0 and not pool._holds_frames() and pool._src == {}


def test_sources_up_to_the_model_area_are_accepted(lr):
    pool = LivePool(lr, 3, size=(64, 64))
    hs = [pool.open() for _ in range(3)]
    pool.push(dict(zip(hs, [np.zeros(s + (3,), np.uint8) for s in ((64, 64), (128, 32), (1, 4096))])))
    assert [pool._src[pool._streams[h][0]] for h in hs] == [(64, 64), (128, 32), (1, 4096)]


def test_video_restorer_has_no_source_limit(monkeypatch):
    """VideoRestorer.stream(size=...) stages whole batches of source frames: a source larger than the model size is
    downscaled, and nothing is rejected before the device."""
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    seen = {}

    class Eng:
        dev = torch.device('cpu')

        def restore_windows(self, frames, idx, **kw):
            seen.update(kw, shape=tuple(frames.shape))
            n = idx.numel() // 3
            return torch.zeros((n,) + kw['size'] + (3,), dtype=torch.uint8)

    class M:
        def engine(self):
            return Eng()
    vr = VideoRestorer(M(), clips_per_batch=4)
    got = np.stack(list(vr.stream(iter(np.zeros((3, 300, 200, 3), np.uint8)), size=[64.0, 128])))
    assert got.shape == (3, 64, 128, 3) and seen['shape'] == (3, 300, 200, 3) and seen['size'] == (64, 128)


# ------------------------------------------------------------------ a pool of source frames on the stub engine
class _LrEngine(_StubEngine):
    """The stub engine, also recording the size table and the staged rgb24 rows of each step."""

    def pool_step(self, u8, x, ring, slots, index, w, adain, out_u8, sizes=None):
        if slots is not None:
            S = u8.shape[0] // 4
            self.calls.append(('sizes', None if sizes is None else sizes.view(-1, 3).tolist(),
                               u8[3 * S:3 * S + slots.numel()].clone()))
        super().pool_step(u8, x, ring, slots, index, w, adain, out_u8)


@pytest.fixture
def lr(stub, monkeypatch):
    resized = []
    monkeypatch.setattr(ops, 'u8hwc_resize_to_f32nchw', lambda x_u8, out, hw, sizes=None: resized.append(hw) or out)
    stub.eng = _LrEngine()
    stub.resized = resized
    return stub


def _src(k, j, hw):
    return np.random.RandomState(100 * k + j).randint(0, 256, hw + (3,), dtype=np.uint8)


@pytest.mark.parametrize('graph', [False, True])
def test_each_step_uploads_the_source_sizes_and_packs_the_rows(lr, graph):
    H, W = 64, 128
    pool = LivePool(lr, 3, size=(H, W), cuda_graph=graph)
    srcs = [(16, 16), (37, 53), (64, 128)]
    hs = [pool.open() for _ in srcs]
    for j in range(2):
        pool.push({h: _src(k, j, hw) for k, (h, hw) in enumerate(zip(hs, srcs))})
        _, table, rows = _steps(lr.eng, 'sizes')[-1]
        assert table == [[h, w, k * H * W * 3] for k, (h, w) in enumerate(srcs)]
        for k, (h, w) in enumerate(srcs):
            assert np.array_equal(rows[k].view(-1)[:h * w * 3].numpy(), _src(k, j, (h, w)).reshape(-1))
    pool.push({hs[2]: _src(2, 2, srcs[2])})                     # one stream: its row is staging row 0
    assert _steps(lr.eng, 'sizes')[-1][1] == [[64, 128, 0]]
    out = pool.flush(hs[0])
    assert out.shape == (H, W, 3)


def test_model_size_pools_stage_as_before(lr):
    pool = LivePool(lr, 2)
    a = pool.open()
    pool.push({a: np.zeros((64, 64, 3), np.uint8)})
    assert _steps(lr.eng, 'sizes')[-1][1] is None and pool._state.idx.numel() == 10 * 2 and not pool._state.lr


def test_source_size_changes_are_per_stream(lr):
    pool = LivePool(lr, 2, size=(64, 64))
    a, b = pool.open(), pool.open()
    pool.push({a: _src(0, 0, (16, 16)), b: _src(1, 0, (32, 48))})
    n = len(lr.eng.calls)
    with pytest.raises(ValueError, match='changed'):
        pool.push({a: _src(0, 1, (32, 48)), b: _src(1, 1, (32, 48))})
    assert len(lr.eng.calls) == n and [pool._streams[h][1] for h in (a, b)] == [1, 1]
    pool.push({a: _src(0, 1, (16, 16)), b: _src(1, 1, (32, 48))})
    pool.flush(a)
    c = pool.open()                                              # a's rows, a new source size
    pool.push({c: _src(2, 0, (64, 64)), b: _src(1, 2, (32, 48))})
    assert _steps(lr.eng, 'sizes')[-1][1] == [[64, 64, 0], [32, 48, 64 * 64 * 3]]
    live = LiveRestorer(lr, size=(64, 64), cuda_graph=False)
    live.push(_src(0, 0, (8, 8)))
    with pytest.raises(ValueError, match='changed'):
        live.push(_src(0, 1, (8, 16)))
    live.flush()
    live.push(_src(0, 0, (8, 16)))                               # a new stream, a new size


def test_graph_keys_do_not_depend_on_source_sizes(lr):
    pool = LivePool(lr, 2, size=(64, 64))
    a, b = pool.open(), pool.open()
    for j in range(3):
        pool.push({a: _src(0, j, (16, 16)), b: _src(1, j, (40, 24))})
    pool.flush(a)
    assert list(pool._state.graphs) == [(2, 0), (2, 2), (0, 1)] and len(lr.eng.rings) == 1


def test_a_rebuild_upsamples_each_streams_rows_again(lr):
    pool = LivePool(lr, 2, w=0.0, size=(64, 64))
    a, b = pool.open(), pool.open()
    for j in range(2):
        pool.push({a: _src(0, j, (16, 16)), b: _src(1, j, (40, 24))})
    assert lr.resized == []
    pool.configure(b, w=1.0)                                     # the ring gains the skip tensors
    n = len(lr.eng.calls)
    pool.push({a: _src(0, 2, (16, 16)), b: _src(1, 2, (40, 24))})
    assert lr.eng.rings == [False, True]
    assert lr.resized == [(16, 16), (16, 16), (40, 24), (40, 24)]
    assert [c[1] for c in lr.eng.calls[n:] if c[0] == 'frame_step'][:4] == [0, 1, 3, 4]
