"""The live restorer (pgtformer_b200/video.py::LiveRestorer) on the GPU: every output byte equal to the reference's
one-window-per-call loop (oracle/video_oracle.py) and to VideoRestorer.restore, eager and replayed from CUDA graphs;
a replayed step launches nothing through the C ABI; the per-frame work runs once per frame; sessions with different w
share one model; and new weights reach the next step.  VideoRestorer(cuda_graph=True) against eager."""
import numpy as np
import pytest
import torch

from oracle import video_oracle as VO

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


def _frames(n, H, W, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(n, H, W, 3), dtype=np.uint8)


def _reference_loop(model, frames, w, adain):
    def apply_window(win):                       # apply_net_to_frames, inference.py:12-19, on this repo's model
        x = torch.from_numpy(VO.rgbnp2tensor(win)).cuda()
        with torch.no_grad():
            mid = model(x, w=w, adain=adain)[0][1]
        return VO.tensor2rgb(mid.float().cpu().numpy())
    return np.stack(VO.restore_frames(list(frames), apply_window))


def _live(live, frames):
    got = [live.push(f) for f in frames]
    assert got[0] is None and all(g is not None for g in got[1:])
    got = got[1:] + [live.flush()]
    return np.stack(got)


def _same(got, ref):
    assert got.shape == ref.shape and got.dtype == np.uint8
    assert np.array_equal(got, ref), 'max |d| = %d' % np.abs(got.astype(int) - ref.astype(int)).max()


@pytest.mark.parametrize('n,H,W,w,adain', [
    (1, 64, 64, 1.0, True), (2, 64, 64, 1.0, True), (3, 64, 64, 1.0, True), (7, 64, 64, 1.0, True),
    (11, 64, 64, 1.0, True), (5, 64, 64, 0.0, True), (5, 64, 64, 1.0, False), (5, 64, 64, 0.0, False),
    (4, 128, 192, 1.0, True), (3, 512, 512, 1.0, True)])
def test_live_equals_reference_loop_and_video_restorer(model, n, H, W, w, adain):
    from pgtformer_b200.video import LiveRestorer, VideoRestorer
    frames = _frames(n, H, W, 300 + n + H)
    ref = _reference_loop(model, frames, w, adain)
    _same(VideoRestorer(model, w=w, adain=adain, clips_per_batch=4).restore(frames), ref)
    for graph in (False, True):
        live = LiveRestorer(model, w=w, adain=adain, cuda_graph=graph)
        _same(_live(live, frames), ref)
        _same(_live(live, frames), ref)                           # a second stream after flush()
        _same(np.stack(list(live.stream(torch.from_numpy(frames).cuda()))), ref)   # CUDA frames, stream()


def test_graphed_step_launches_nothing(model):
    from pgtformer_b200 import ops
    from pgtformer_b200.video import LiveRestorer
    frames = _frames(9, 64, 64, 5)
    ref = _reference_loop(model, frames, 1.0, True)
    live = LiveRestorer(model)
    got = [live.push(f) for f in frames[:5]]                      # every steady phase captured
    for i in range(5, 9):
        n = ops.launch_count()
        got.append(live.push(frames[i]))
        assert ops.launch_count() == n
    got.append(live.flush())
    _same(np.stack(got[1:]), ref)


def test_per_frame_work_runs_once_per_frame(model):
    from pgtformer_b200.video import LiveRestorer
    eng = model.engine()
    calls = []
    parse_pos = eng.parse_pos
    eng.parse_pos = lambda *a, **k: calls.append(1) or parse_pos(*a, **k)
    try:
        live = LiveRestorer(model, cuda_graph=False)
        for n in (7, 4):
            calls.clear()
            _live(live, _frames(n, 64, 64, n))
            assert len(calls) == n + (1 if n == 7 else 0)             # + the run that sizes a new session's ring
    finally:
        del eng.parse_pos


@pytest.mark.parametrize('graph', [False, True])
def test_sessions_with_different_w_interleave(model, graph):
    from pgtformer_b200.video import LiveRestorer
    a_frames, b_frames = _frames(6, 64, 64, 41), _frames(6, 64, 64, 42)
    refs = _reference_loop(model, a_frames, 1.0, True), _reference_loop(model, b_frames, 0.0, False)
    lives = LiveRestorer(model, w=1.0, cuda_graph=graph), LiveRestorer(model, w=0.0, adain=False, cuda_graph=graph)
    got = ([], [])
    for fa, fb in zip(a_frames, b_frames):
        for k, f in enumerate((fa, fb)):
            r = lives[k].push(f)
            if r is not None:
                got[k].append(r)
    for k in range(2):
        got[k].append(lives[k].flush())
        _same(np.stack(got[k]), refs[k])


@pytest.mark.parametrize('graph', [False, True])
def test_new_weights_reach_the_next_step(network_g, graph):
    """load_state_dict() in the middle of a stream: every frame restored after it comes from the new weights, the frames
    still in the window included."""
    from archs.pgtformer_arch import PGTFormer
    from pgtformer_b200.video import LiveRestorer
    kw = dict(network_g)
    kw.pop('type', None)
    m = PGTFormer(**kw).cuda().eval()
    m.cuda_graph = False
    frames = _frames(6, 64, 64, 77)
    old_ref = _reference_loop(m, frames, 1.0, True)
    live = LiveRestorer(m, cuda_graph=graph)
    got = [live.push(f) for f in frames[:3]][1:]                  # frames 0, 1 on the old weights
    sd = {k: v * 0.9 if v.is_floating_point() else v for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    got += [live.push(f) for f in frames[3:]] + [live.flush()]   # frames 2..5 on the new ones
    new_ref = _reference_loop(m, frames, 1.0, True)
    assert not np.array_equal(old_ref[2:], new_ref[2:])
    _same(np.stack(got[:2]), old_ref[:2])
    _same(np.stack(got[2:]), new_ref[2:])


@pytest.mark.parametrize('reuse', [True, False])
def test_video_restorer_graphed_equals_eager(model, reuse):
    from pgtformer_b200.video import VideoRestorer
    frames = _frames(11, 64, 64, 9)                                # batches of 4, 4 and a ragged 3
    eager = VideoRestorer(model, clips_per_batch=4, reuse_frames=reuse).restore(frames)
    vr = VideoRestorer(model, clips_per_batch=4, reuse_frames=reuse, cuda_graph=True)
    _same(vr.restore(frames), eager)
    _same(vr.restore(frames), eager)                               # replayed
    _same(np.stack(list(vr.stream(iter(frames)))), eager)
