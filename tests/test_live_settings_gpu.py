"""Per-stream settings of a live pool on the GPU: the per-frame SFT weight of the conv epilogues and the per-frame
AdaIN kernel against fp64 (and, for uniform settings, bit for bit against the scalar kernels), every stream of a pool
with mixed w and AdaIN byte for byte what VideoRestorer.restore gives on that stream alone at its settings, settings
changed mid-stream (including the ring rebuilt with and without the SFT skip tensors), and a steady mixed pool that
replays one graph per step shape."""
import hashlib
import re

import numpy as np
import pytest
import torch

from test_gemm_epilogue_gpu import launches
from test_live_pool_cpu import _schedule
from test_live_pool_gpu import _same, _video, model  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
DEV = 'cuda'


# ------------------------------------------------------------------ the per-frame SFT weight
def _rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale)


# (F, H, W, Cin, Cout, out dtype, scale view offset, the launch the library must pick)
SFT_CASES = [
    (3, 32, 32, 64, 256, 'bf16', 0, r'^conv3 .* BN128 t1x4x32 e1$'),       # GEMM / conv kernel, TMA-store epilogue
    (3, 32, 32, 128, 512, 'bf16', 0, r'^conv3 .* BN128 t1x4x32 e1$'),
    (3, 8, 8, 64, 64, 'bf16', 0, r'^conv3 .* BN64 t2x8x8 e1$'),             # tiles of two frames, F % 2 != 0
    (3, 32, 32, 64, 256, 'f32', 0, r'^conv3 .* BN128 t1x4x32 e0$'),         # direct per-thread path
    (3, 32, 32, 64, 256, 'bf16', 1, r'^conv3 .* BN128 t1x4x32 e0$'),        # misaligned scale view: direct path
    (4, 16, 16, 64, 128, 'bf16', 0, r'^halo3 .* BN128 e1 r0$'),             # halo conv, TMA-store epilogue
    (3, 24, 40, 64, 64, 'bf16', 0, r'^halo3 .* BN64 e1 r1$'),
    (3, 16, 16, 64, 128, 'f32', 0, r'^halo3 .* BN128 e0 r0$'),              # halo conv, direct path
]


def _sft_inputs(F, H, W, Cin, Cout, aoff, seed):
    from pgtformer_b200.engine import _pack_conv
    x = _rnd((F, H, W, Cin), seed).to(torch.bfloat16)
    w = _rnd((Cout, Cin, 3, 3), seed + 1, 0.05)
    b = _rnd((Cout,), seed + 2, 0.1)
    res = _rnd((F, H, W, Cout), seed + 3).to(torch.bfloat16)
    scale = _rnd((F, H, W, Cout + aoff), seed + 4).to(torch.bfloat16)
    return x, w, b, res, scale, _pack_conv(w.to(DEV))


def _sft_run(x, wp, b, res, scale, Cout, aoff, out_dtype, wgt):
    from pgtformer_b200 import ops
    F, H, W, _ = x.shape
    out = torch.empty(F, H, W, Cout, dtype=out_dtype, device=DEV)
    sc = scale.to(DEV)[..., aoff:]
    ops.conv(x.to(DEV), wp, Cout, out, bias=b.to(DEV), residual=res.to(DEV), sft_scale=sc, sft_w=wgt)
    return out


@pytest.mark.parametrize('F,H,W,Cin,Cout,odt,aoff,path', SFT_CASES)
def test_per_frame_sft_weight_against_fp64(F, H, W, Cin, Cout, odt, aoff, path, tmp_path):
    """y = r + w[f] (r s + conv(x) + b) per output frame f, frames with w = 0 included; every element within the
    bf16 rounding of its magnitude bound of the fp64 result."""
    x, w, b, res, scale, wp = _sft_inputs(F, H, W, Cin, Cout, aoff, F * H + Cout)
    wf = torch.tensor([0.0, 0.7, 1.3, 0.25][:F], dtype=torch.float32, device=DEV)
    dt = torch.bfloat16 if odt == 'bf16' else torch.float32
    out = None

    def run():
        nonlocal out
        out = _sft_run(x, wp, b, res, scale, Cout, aoff, dt, wf)
    descs = launches(run, tmp_path)
    assert len(descs) == 1 and re.search(path, descs[0]), descs
    x64, w64 = x.double().permute(0, 3, 1, 2), w.to(torch.bfloat16).double()
    z = torch.nn.functional.conv2d(x64, w64, b.double(), padding=1).permute(0, 2, 3, 1)
    za = torch.nn.functional.conv2d(x64.abs(), w64.abs(), b.double().abs(), padding=1).permute(0, 2, 3, 1)
    r, s = res.double(), scale.double()[..., aoff:]
    wv = wf.double().cpu().view(F, 1, 1, 1)
    ref = r + wv * (r * s + z)
    bound = r.abs() + wv.abs() * ((r * s).abs() + za)
    err = (out.double().cpu() - ref).abs()
    assert (err <= bound * 2.0 ** -8 + 1e-30).all(), float((err / bound.clamp_min(1e-30)).max())
    assert torch.equal(out[0].cpu(), res[0].to(dt))          # w = 0: the residual itself


@pytest.mark.parametrize('F,H,W,Cin,Cout,odt,aoff,path', SFT_CASES)
def test_uniform_per_frame_weights_equal_the_scalar_path_bit_for_bit(F, H, W, Cin, Cout, odt, aoff, path):
    x, w, b, res, scale, wp = _sft_inputs(F, H, W, Cin, Cout, aoff, F * W + Cout)
    dt = torch.bfloat16 if odt == 'bf16' else torch.float32
    for v in (0.0, 0.3, 1.0):
        wf = torch.full((F,), v, dtype=torch.float32, device=DEV)
        a = _sft_run(x, wp, b, res, scale, Cout, aoff, dt, wf)
        c = _sft_run(x, wp, b, res, scale, Cout, aoff, dt, v)
        assert torch.equal(a.view(torch.int16 if odt == 'bf16' else torch.int32),
                           c.view(torch.int16 if odt == 'bf16' else torch.int32)), v
    # and each frame of a mixed vector as the scalar path at that frame's weight
    wf = torch.tensor([0.5, 0.0, 1.0, 0.3][:F], dtype=torch.float32, device=DEV)
    a = _sft_run(x, wp, b, res, scale, Cout, aoff, dt, wf)
    for f in range(F):
        c = _sft_run(x, wp, b, res, scale, Cout, aoff, dt, float(wf[f]))
        assert torch.equal(a[f], c[f]), f


def test_per_frame_weights_are_rejected_on_a_gemm():
    from pgtformer_b200 import ops
    a = torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV)
    wt = torch.zeros(64, 64, dtype=torch.bfloat16, device=DEV)
    out = torch.empty(128, 64, dtype=torch.bfloat16, device=DEV)
    ep = ops.make_epilogue(out, residual=out, sft_scale=out, sft_w=torch.ones(1, device=DEV))
    lib = ops.L.load()
    import ctypes
    assert lib.pgt_linear_bf16(ops._p(a), 64, ops._p(wt), 64, 128, 64, 64, ctypes.byref(ep), ops._stream()) == -1


# ------------------------------------------------------------------ the per-frame AdaIN
@pytest.mark.parametrize('qdt', [torch.float32, torch.bfloat16])
def test_adain_flags_against_fp64_and_the_scalar_kernels(qdt):
    from pgtformer_b200 import ops, torch_ops
    F, HW, C = 4, 256, 256
    q = (_rnd((F, HW, C), 5) * 3 + 1).to(qdt).to(DEV)
    lq = (_rnd((F, HW, C), 6) * 0.5 - 2).to(torch.bfloat16).to(DEV)
    flags = torch.tensor([1, 0, 0, 1], dtype=torch.int32, device=DEV)
    got = ops.adain(q, lq, torch.empty(F, HW, C, dtype=torch.bfloat16, device=DEV), flags=flags)
    on = ops.adain(q, lq, torch.empty(F, HW, C, dtype=torch.bfloat16, device=DEV))
    for f in (0, 3):                                              # flag on: AdaIN, the bits of pgt_adain
        assert torch.equal(got[f].view(torch.int16), on[f].view(torch.int16)), f
        qd, ld = q[f].double(), lq[f].double()
        ref = (qd - qd.mean(0)) / (qd.var(0) + 1e-5).sqrt() * (ld.var(0) + 1e-5).sqrt() + ld.mean(0)
        assert ((got[f].double() - ref).abs() <= ref.abs() * 2.0 ** -8 + 1e-4).all()
    for f in (1, 2):                                              # flag off: the bf16 rounding of q
        assert torch.equal(got[f].view(torch.int16), q[f].to(torch.bfloat16).view(torch.int16)), f
    shim = torch.empty_like(got)
    torch_ops.load().adain_frames(q, lq, flags, 1e-5, shim)
    assert torch.equal(shim.view(torch.int16), got.view(torch.int16))
    ones = torch.ones(F, dtype=torch.int32, device=DEV)
    allon = ops.adain(q, lq, torch.empty_like(got), flags=ones)
    assert torch.equal(allon.view(torch.int16), on.view(torch.int16))


# ------------------------------------------------------------------ streams against VideoRestorer
SETTINGS = [(w, a) for w in (0.0, 0.3, 0.5, 1.0) for a in (True, False)]

CASES = [  # (H, W, lengths, max_streams, seed)
    (64, 64, [1, 2, 3, 5, 7, 11], 6, 0),
    (64, 64, [6, 2, 4, 5, 3], 3, 1),
    (64, 64, [4, 3], 1, 2),
    (128, 192, [5, 3, 7, 4], 4, 3),
    (512, 512, [3, 4, 2], 3, 4),
]

_refs = {}


def _restore_alone(model, video, w, adain):  # noqa: F811
    """VideoRestorer.restore of one stream at its settings (each video and setting restored once per session)."""
    from pgtformer_b200.video import VideoRestorer
    key = (hashlib.sha1(video.tobytes()).hexdigest(), video.shape, w, adain)
    if key not in _refs:
        _refs[key] = VideoRestorer(model, w=w, adain=adain, clips_per_batch=4).restore(video)
    return _refs[key]


def _play(pool, ops, videos, conf):
    """Plays a schedule; each stream opens with its settings conf[k] -> {stream: restored frames}."""
    handles, got, pushed = {}, {}, {}
    for op, arg in ops:
        if op == 'open':
            handles[arg], got[arg], pushed[arg] = pool.open(*conf[arg]), [], 0
        elif op == 'flush':
            got[arg].append(pool.flush(handles.pop(arg)))
        else:
            res = pool.push({handles[k]: videos[k][pushed[k]] for k in arg})
            for k in arg:
                if pushed[k]:
                    got[k].append(res[handles[k]])
                pushed[k] += 1
    return {k: np.stack(v) for k, v in got.items()}


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('H,W,lengths,S,seed', CASES)
def test_mixed_settings_equal_video_restorer_alone(model, H, W, lengths, S, seed, graph):  # noqa: F811
    from pgtformer_b200.video import LivePool
    rnd = np.random.RandomState(seed)
    conf = [SETTINGS[i] for i in rnd.permutation(len(SETTINGS))[:len(lengths)]]
    videos = [_video(n, H, W, 300 + 10 * seed + k) for k, n in enumerate(lengths)]
    pool = LivePool(model, S, cuda_graph=graph)
    got = _play(pool, _schedule(seed, lengths, S), videos, conf)
    for k, v in enumerate(videos):
        _same(got[k], _restore_alone(model, v, *conf[k]))


@pytest.mark.parametrize('graph', [False, True])
def test_settings_changed_mid_stream(model, graph):  # noqa: F811
    """Two streams start at w = 0; one goes to w = 1 (the ring is rebuilt with the SFT skip tensors), later back to 0
    with AdaIN off while the other turns AdaIN on, then to w = 0.5.  Each frame equals VideoRestorer at the settings in
    force when it was returned."""
    from pgtformer_b200.video import LivePool, LiveRestorer
    videos = [_video(8, 64, 64, 500), _video(7, 64, 64, 501)]
    # (step, stream, w, adain): configure before that step's push
    changes = {3: [(0, 1.0, True)], 5: [(0, 0.0, False), (1, None, True)], 6: [(1, 0.5, None)]}
    conf = [[0.0, True], [0.0, False]]
    pool = LivePool(model, 2, w=0.0, cuda_graph=graph)
    hs = [pool.open(w=0.0, adain=True), pool.open(w=0.0, adain=False)]
    got, used, rings = [[], []], [[], []], []
    for step in range(9):
        for k, w, a in changes.get(step, []):
            pool.configure(hs[k], w=w, adain=a)
            conf[k] = [w if w is not None else conf[k][0], a if a is not None else conf[k][1]]
        frames = {hs[k]: v[step] for k, v in enumerate(videos) if step < len(v)}
        res = pool.push(frames) if frames else {}
        for k, v in enumerate(videos):
            if step == len(v):
                res[hs[k]] = pool.flush(hs[k])
            if res.get(hs[k]) is not None:
                got[k].append(res[hs[k]])
                used[k].append(tuple(conf[k]))
        rings.append(bool(pool._state.ring['feats']) if pool._state is not None else None)
    assert rings[:3] == [False] * 3 and rings[3:] == [True] * 6
    for k, v in enumerate(videos):
        assert len(got[k]) == len(v)
        for i, (f, c) in enumerate(zip(got[k], used[k])):
            _same(f, _restore_alone(model, v, *c)[i])
    live = LiveRestorer(model, w=0.0, adain=False, cuda_graph=graph)   # the same on a restorer of one stream
    out = [live.push(f) for f in videos[1][:3]][1:]
    live.configure(w=1.0, adain=True)
    out += [live.push(f) for f in videos[1][3:]] + [live.flush()]
    for i, f in enumerate(out):
        _same(f, _restore_alone(model, videos[1], *((0.0, False) if i < 2 else (1.0, True)))[i])


def test_steady_mixed_pool_replays_one_graph_per_step_shape(model):  # noqa: F811
    from pgtformer_b200 import ops
    from pgtformer_b200.video import LivePool
    S, n = 4, 8
    conf = [(1.0, True), (0.0, True), (0.5, False), (0.0, False)]
    videos = [_video(n, 64, 64, 700 + k) for k in range(S)]
    pool = LivePool(model, S)
    hs = [pool.open(*c) for c in conf]
    got = [[] for _ in range(S)]
    for j in range(n):
        if j == 3:
            keys = set(pool._state.graphs)
            assert keys == {(S, 0), (S, S, 2)}
            replays = []
            for key, g in pool._state.graphs.items():
                g.replay = (lambda r, key: lambda: replays.append(key) or r())(g.replay, key)
            launches_before = ops.launch_count()
        res = pool.push({h: videos[k][j] for k, h in enumerate(hs)})
        for k, h in enumerate(hs):
            if res[h] is not None:
                got[k].append(res[h])
    assert ops.launch_count() == launches_before and set(pool._state.graphs) == keys
    assert replays == [(S, S, 2)] * (n - 3)
    for k, h in enumerate(hs):
        got[k].append(pool.flush(h))
        _same(np.stack(got[k]), _restore_alone(model, videos[k], *conf[k]))
