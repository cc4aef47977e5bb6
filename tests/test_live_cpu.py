"""Host logic of the live restorer (pgtformer_b200/video.py::LiveRestorer): its push / flush schedule against the
reference's window loop, and the frame checks that run before any device work."""
import inspect

import numpy as np
import pytest
import torch

from pgtformer_b200.video import LiveRestorer, VideoRestorer, window_indices


class _NoDevice:
    """A model stand-in whose engine must never be reached."""

    def __init__(self):
        self.engine_calls = 0

    def parameters(self):
        yield torch.zeros(1)

    def engine(self):
        self.engine_calls += 1
        raise AssertionError('device work started')


def _recording(model=None):
    """A LiveRestorer whose device step returns the frame indices of the window it would restore."""
    live = LiveRestorer(model or _NoDevice())
    live.steps = []

    def step(t, n, new, win):
        live.steps.append((n, new, win))
        return win
    live._step = step
    return live


def _frames(n, hw=(64, 128)):
    return [np.full(hw + (3,), i % 256, np.uint8) for i in range(n)]


@pytest.mark.parametrize('n', range(1, 13))
def test_push_flush_schedule_is_the_reference_window_loop(n):
    live = _recording()
    for rnd in range(2):                                      # and again after the reset that flush() makes
        got = [live.push(f) for f in _frames(n)]
        assert got[0] is None
        got = got[1:] + [live.flush()]
        assert got == window_indices(n), rnd
        # each frame goes into the ring once, into slot frame % 3, when it is pushed
        assert [(s[0], s[1]) for s in live.steps if s[1] is not None] == [(i, i % 3) for i in range(n)]
        live.steps.clear()
    assert live.flush() is None                               # an empty stream restores nothing


@pytest.mark.parametrize('n', [0, 1, 2, 5])
def test_stream_yields_every_frame_once(n):
    live = _recording()
    assert list(live.stream(iter(_frames(n)))) == window_indices(n)
    assert list(live.stream(iter(_frames(n, (128, 64))))) == window_indices(n)   # a new stream may change the size


@pytest.mark.parametrize('frame', [
    np.zeros((64, 64, 3), np.float32),                        # dtype
    np.zeros((64, 64, 3), np.int8),
    torch.zeros(64, 64, 3, dtype=torch.int32),
    np.zeros((1, 64, 64, 3), np.uint8),                       # rank
    np.zeros((64, 64), np.uint8),
    np.zeros((64, 64, 4), np.uint8),                          # not rgb24
    np.zeros((3, 64, 64), np.uint8),
    np.zeros((96, 64, 3), np.uint8),                          # not multiples of 64
    torch.zeros(64, 100, 3, dtype=torch.uint8),
    np.zeros((0, 64, 3), np.uint8),
])
def test_bad_frames_raise_before_any_device_work(frame):
    model = _NoDevice()
    live = LiveRestorer(model)
    with pytest.raises(ValueError):
        live.push(frame)
    assert model.engine_calls == 0


def test_size_change_inside_a_stream_raises_before_any_device_work():
    live = _recording()
    live.push(np.zeros((64, 64, 3), np.uint8))
    with pytest.raises(ValueError, match='changed'):
        live.push(np.zeros((64, 128, 3), np.uint8))
    assert len(live.steps) == 1
    assert live.push(np.zeros((64, 64, 3), np.uint8)) == (0, 0, 1)     # the stream goes on at its own size


def test_cpu_model_raises_the_no_cpu_path_error(network_g):
    from archs.pgtformer_arch import PGTFormer
    kw = dict(network_g)
    kw.pop('type', None)
    live = LiveRestorer(PGTFormer(**kw))
    with pytest.raises(RuntimeError, match='no CPU path'):
        live.push(np.zeros((64, 64, 3), np.uint8))


def test_video_restorer_defaults_are_unchanged():
    p = inspect.signature(VideoRestorer).parameters
    assert {k: v.default for k, v in p.items() if k != 'model'} == dict(
        w=1.0, adain=True, clips_per_batch=16, reuse_frames=True, cuda_graph=False)
    vr = VideoRestorer(model=None)
    assert (vr.w, vr.adain, vr.clips_per_batch, vr.reuse_frames, vr.cuda_graph) == (1.0, True, 16, True, False)
