"""The launch sequences of the six registered models' engines, run on the CPU with every kernel call replaced by a
recorder that returns its output argument, checked against the rule the block walker (Engine._walk) states.

Invariants, for every call of every model:
- every GroupNorm that takes fused statistics (groupnorm_apply_stats, groupnorm_ab with stats) takes, frame by frame,
  the ones the producer of that very tensor wrote in its epilogue (or their frame gather, on the streaming and live
  paths, which gather frames and statistics from a batch of distinct frames or from a live ring's slots);
- a GroupNorm whose input came straight from a conv, linear, conv_rgb, conv_up2x or swin_mlp launch computes its own
  statistics (groupnorm_silu, groupnorm_ab without stats) only where that producer could not have fused them: a tile
  grid that does not divide the frame (conv_tiles_exact), a channel count gn_stats_supported rejects, a non-contiguous
  output, H*W not a multiple of 128 for a linear, swin_mlp or conv_in, a conv_in width other than 64 or 128.  A concat
  buffer written in slices has no single producer and is never such an input."""
import contextlib
import copy
import inspect
import itertools

import pytest
import torch

from test_pack_cpu import packed

# the kernel calls the engines make at run time
OPS = ('linear', 'conv', 'conv_rgb', 'conv_up2x', 'groupnorm_silu', 'groupnorm_apply_stats', 'groupnorm_ab',
       'conv_out_gn', 'layernorm', 'ln_linear', 'swin_mlp', 'window_attention', 'window_attention_tc',
       'window3d_attention', 'mha', 'argmax_gather', 'l2_argmin_tc', 'l2_argmin_tc_split', 'soft_codes', 'sample_codes',
       'rq_residual', 'rq_embed', 'vq_stats', 'adain', 'maxpool3x3s2', 'global_avgpool', 'channel_affine',
       'assemble_cond', 'gather_frames', 'copy2d', 'regroup_frames', 'f32nchw_to_u8hwc')
# what a call returns, where that is not its `out` argument
RETURNS = {'argmax_gather': ('idx_out', 'quant'), 'l2_argmin_tc': ('idx_out', 'quant'),
           'l2_argmin_tc_split': ('idx_out', 'quant'), 'groupnorm_ab': 'ab', 'rq_residual': 'agg',
           'vq_stats': 'scalars', 'assemble_cond': 'cond', 'sample_codes': 'idx_out', 'f32nchw_to_u8hwc': 'out_u8'}


def _key(t):
    return t.data_ptr(), tuple(t.shape), t.stride()


def _frames(t, n):
    """(address, shape, strides) of each of the n frames of t along its first dimension; a tensor whose first dimension
    is not n (a flat statistics buffer) splits into n equal flat parts."""
    if t.dim() > 1 and t.shape[0] == n:
        step, shape, stride = t.stride(0), tuple(t.shape[1:]), t.stride()[1:]
    else:
        step = t.numel() // n
        shape, stride = (step,), (1,)
    return [(t.data_ptr() + f * step * t.element_size(), shape, stride) for f in range(n)]


class Recorder:
    """Replaces the ops kernel calls.  `log` holds one (op, tensor shapes, writes statistics, reads statistics) entry
    per call; `violations` the calls that break an invariant."""

    def __init__(self, ops):
        self.ops = ops
        self.log, self.violations = [], []
        # data_ptr -> (key of the tensor last written there, op, whether that op could have fused the next GroupNorm's
        # statistics); a write into a slice that starts there replaces the entry of the whole buffer
        self.producer = {}
        # frame (_frames) -> what the last write there left: a token of that write, or ('stats', token) for the
        # GroupNorm statistics of the frame that holds that token; a frame gather moves both with the frames
        self.held = {}
        self.tokens = itertools.count()

    def could_fuse(self, name, a):
        out = a['out']
        if out.dim() != 4 or out.dtype != torch.bfloat16 or not out.is_contiguous() or \
                not self.ops.gn_stats_supported(out.shape[-1]):
            return False
        if name == 'conv':
            if a['nchw']:
                return False
            _, H, W, _ = a['x'].shape
            return self.ops.conv_tiles_exact(H, W, a['cout'], a['ksize'], a['stride'], a['pad_lo']) > 0
        if name == 'conv_up2x':
            _, H, W, _ = a['x'].shape
            return self.ops.conv_tiles_exact(H, W, a['cout'], 2, 1, 1) > 0
        hw = out.shape[1] * out.shape[2] % 128 == 0
        if name == 'conv_rgb':
            return hw and a['ksize'] == 3 and out.shape[-1] in (64, 128)
        return hw                                   # linear, swin_mlp

    def call(self, name, a):
        gn_in = a.get('stats') if name in ('groupnorm_apply_stats', 'groupnorm_ab') else None
        writes = a.get('gn_stats') is not None
        self.log.append((name, tuple(tuple(v.shape) for v in a.values() if torch.is_tensor(v)), writes,
                         gn_in is not None))
        x = a.get('x')
        if name in ('groupnorm_apply_stats', 'groupnorm_ab') and gn_in is not None:
            want = [('stats', self.held.get(k)) for k in _frames(x, x.shape[0])]
            if any(w[1] is None for w in want) or [self.held.get(k) for k in _frames(gn_in, x.shape[0])] != want:
                self.violations.append('%s on %s reads statistics of another tensor' % (name, tuple(x.shape)))
        elif name in ('groupnorm_silu', 'groupnorm_ab'):
            key, op, fusable = self.producer.get(x.data_ptr(), (None, None, False))
            if fusable and key == _key(x):
                self.violations.append('%s recomputes the statistics of a %s output %s that could have fused them'
                                       % (name, op, tuple(x.shape)))
        out = a.get('out')
        if torch.is_tensor(out):
            fusable = name in ('conv', 'linear', 'conv_rgb', 'conv_up2x', 'swin_mlp') and self.could_fuse(name, a)
            self.producer[out.data_ptr()] = (_key(out), name, fusable)
            frames = _frames(out, out.shape[0])
            if name == 'gather_frames':
                src = _frames(x, x.shape[0])
                for k, i in zip(frames, a['idx_i32'].tolist()):
                    self.held[k] = self.held.get(src[i], ('unknown', next(self.tokens)))
            else:
                for k in frames:
                    self.held[k] = next(self.tokens)
            if writes:
                for k, s in zip(frames, _frames(a['gn_stats'], out.shape[0])):
                    self.held[s] = ('stats', self.held[k])


def install(monkeypatch):
    """A Recorder in place of the ops kernel calls."""
    from pgtformer_b200 import ops
    rec = Recorder(ops)

    def fake(name):
        sig = inspect.signature(getattr(ops, name))

        def run(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            a = b.arguments
            rec.call(name, a)
            ret = RETURNS.get(name, 'out')
            return tuple(a[r] for r in ret) if isinstance(ret, tuple) else a[ret]
        return run

    for name in OPS:
        monkeypatch.setattr(ops, name, fake(name))
    monkeypatch.setattr(ops, 'codebook_pack', lambda cb, K: (torch.empty(K, cb.shape[1], dtype=torch.bfloat16),
                                                             torch.empty(K + 2)))
    # the engine's methods select its device for the launches; here there is none
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return rec


@pytest.fixture
def recorder(monkeypatch):
    return install(monkeypatch)


_engines = {}


def _engine(name, network_g):
    """One engine per model on the CPU (Engine._repack of the synthetic state dict), built on first use."""
    if name not in _engines:
        if name == 'TDCRQVAE3_r2':                   # two res blocks per level
            g = copy.deepcopy(network_g)
            g['ddconfig']['num_res_blocks'] = 2
            _engines[name] = packed('PGTFormer', g)[0]
        else:
            _engines[name] = packed('PGTFormer' if name == 'TDCRQVAE3' else name, network_g)[0]
    return _engines[name]


def _x(*shape):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(0))


def _live(eng, H, W, w, n=4):
    """LiveRestorer's schedule on the engine: frame j into ring slot j % 3, then the window of frame j - 1
    (video.window_indices), and the last frame's window at the end.  Four frames reuse slot 0."""
    from pgtformer_b200.video import window_indices
    ring = eng.live_ring(H, W, w)
    out = torch.empty(1, H, W, 3, dtype=torch.uint8)
    wins = window_indices(n)
    for j in range(n + 1):
        if j < n:
            eng.frame_step(_x(1, 3, H, W), j % 3, ring)
        if j > 0:
            eng.window_step(torch.tensor([k % 3 for k in wins[j - 1]], dtype=torch.int32), w, True, ring, out)


def _calls(name, eng, b, H, W):
    """(label, thunk) of every call of `name` the walk is checked on, at b clips / images of H x W."""
    if name == 'PGTFormer':
        x = _x(3 * b, 3, H, W)
        fi = torch.tensor([0, 1, 2] + [1, 2, 3] * (b - 1), dtype=torch.int32)
        return [('w1', lambda: eng.forward(x, w=1.0)), ('w0', lambda: eng.forward(x, w=0.0)),
                ('code_only', lambda: eng.forward(x, code_only=True)),
                ('stream', lambda: eng.forward(_x(2 + b, 3, H, W), w=1.0, frame_index=fi)),
                ('live_w1', lambda: _live(eng, H, W, 1.0)), ('live_w0', lambda: _live(eng, H, W, 0.0))]
    if name.startswith('TDCRQVAE3'):
        x = _x(3 * b, 3, H, W)
        z = _x(3 * b, H // 16, W // 16, eng.arch.embed_dim)
        return [('forward_vq', lambda: eng.forward_vq(x)), ('encode', lambda: eng.encode(x)),
                ('decode', lambda: eng.decode(z))]
    if name == 'TDRQVAE':
        return [('forward', lambda: eng.forward(_x(b, 3 if b == 1 else 7, 3, H, W)))]
    if name.startswith('RQVAE'):
        return [('forward_vq', lambda: eng.forward_vq(_x(b, 3, H, W)))]
    if name == 'VQGAN':
        return [('forward', lambda: eng.forward(_x(b, 3, H, W)))]
    x = _x(b, 3, H, W)
    return [('w0', lambda: eng.forward(x, w=0.0)), ('w05', lambda: eng.forward(x, w=0.5, adain=True))]


# (model, b, H, W): each model's fixture sizes, 64 x 192 where the model takes it, and TDCRQVAE3 with two res blocks
# per level
CASES = [('PGTFormer', 1, 64, 64), ('PGTFormer', 2, 128, 128), ('PGTFormer', 1, 64, 192), ('PGTFormer', 1, 192, 64),
         ('PGTFormer', 2, 64, 128), ('PGTFormer', 1, 512, 512),
         ('TDCRQVAE3', 1, 64, 64), ('TDCRQVAE3', 2, 128, 128), ('TDCRQVAE3', 1, 64, 192),
         ('TDCRQVAE3_r2', 1, 64, 64), ('TDCRQVAE3_r2', 1, 128, 128), ('TDCRQVAE3_r2', 1, 64, 192),
         ('TDRQVAE', 1, 64, 64), ('TDRQVAE', 2, 128, 128), ('TDRQVAE', 1, 64, 192), ('TDRQVAE', 1, 512, 512),
         ('RQVAE_r1', 1, 256, 256), ('RQVAE_r1', 2, 256, 256), ('RQVAE_r2', 2, 128, 128), ('RQVAE_r2', 1, 128, 256),
         ('RQVAE_r2', 2, 96, 160),
         ('VQGAN', 2, 128, 128), ('VQGAN', 1, 256, 384), ('VQGAN', 1, 512, 512),
         ('CodeFormer', 1, 512, 512), ('CodeFormer', 2, 512, 512)]


def record(name, b, H, W, network_g, rec):
    """{label: recorded log} of the calls of `name` at this size."""
    eng = _engine(name, network_g)
    logs = {}
    for label, thunk in _calls(name, eng, b, H, W):
        n = len(rec.log)
        thunk()
        logs[label] = rec.log[n:]
    return logs


@pytest.mark.parametrize('name,b,H,W', CASES)
def test_groupnorm_statistics_follow_the_walk_rule(network_g, recorder, name, b, H, W):
    logs = record(name, b, H, W, network_g, recorder)
    assert not recorder.violations, '\n'.join(recorder.violations[:10])
    for label, log in logs.items():
        assert any(e[0] == 'groupnorm_apply_stats' for e in log), label     # fused statistics are consumed
        assert any(e[0] in ('conv', 'linear') for e in log), label
