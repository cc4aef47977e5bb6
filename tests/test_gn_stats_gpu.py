"""Every GroupNorm statistic an engine takes from a producer's epilogue, checked against the tensor it normalises.

Most GroupNorms in the encoders and decoders do not read their input for statistics: the epilogue of the conv or
linear that wrote the tensor already summed it per (frame, 32-row chunk, group) (gemm_tc.cu gn_stats, attached to the
tensor as `_pgt_gn` by Engine._gn_stats), and Engine._gn (groupnorm_apply_stats) and Engine.decoder_out
(groupnorm_ab) trust those sums.  Here both consumers are wrapped: before the kernel runs, the buffer's chunks are
summed per frame and group (`stats.view(F, chunks_per_frame, 32, 2).sum(1)`: [frame][tile][quadrant] for convs and
linears, [frame][phase][tile][quadrant] for the upsample conv) and compared with fp64 sums Σx and Σx² of the bf16
tensor x being normalised.  A conv whose 128-pixel tile grid does not divide the frame would add the rows past the
frame's edge (act(bias) of TMA zero-fill) to its sums; every model is therefore run at a power-of-two size and,
where it takes others, at frame sizes some levels' tile grids do not divide.

Bound.  The epilogue sums the fp32 values f before they are rounded to the stored bf16 x, and |x - f| <= 2^-9 |f|
(round to nearest, 8 significant bits), so |f - x| <= 2^-9 (1 - 2^-9)^-1 |x| < 2^-8 |x| and
|f^2 - x^2| = |f - x| |f + x| < 2^-7 x^2.  Per (frame, group) this gives |ΔΣx| <= 2^-8 Σ|x| and |ΔΣx²| <= 2^-7 Σx².
Each chunk partial is an fp32 sum of at most 32 rows x 32 channels = 1024 terms, off by at most 1024 * 2^-24 = 2^-14
of its sum of magnitudes (itself < (1 + 2^-8) times that of x); the chunks are added here in fp64.  So:
|ΔΣx| <= (2^-8 + 2^-13) Σ|x| and |ΔΣx²| <= (2^-7 + 2^-13) Σx², with no slack that depends on the data."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda'

SUM_BOUND = 2.0 ** -8 + 2.0 ** -13
SQ_BOUND = 2.0 ** -7 + 2.0 ** -13


class Audit:
    """Checks the fused statistics each consuming GroupNorm is handed; `norm` is the consumer's weight prefix."""

    def __init__(self):
        self.norm = None
        self.fused = 0
        self.violations = []

    def check(self, x, stats, chunks_per_frame):
        self.fused += 1
        Fr, H, W, C = x.shape
        assert stats.numel() == Fr * chunks_per_frame * 64, (self.norm, stats.numel(), Fr, chunks_per_frame)
        got = stats.view(Fr, chunks_per_frame, 32, 2).double().sum(1)
        v = x.double().reshape(Fr, H * W, 32, C // 32)
        s, a, q = v.sum((1, 3)), v.abs().sum((1, 3)), v.pow(2).sum((1, 3))
        for k, (ref, allowed) in enumerate(((s, SUM_BOUND * a), (q, SQ_BOUND * q))):
            ratio = ((got[..., k] - ref).abs() / allowed.clamp_min(1e-300)).max().item()
            if ratio > 1.0:
                self.violations.append('%s [%d, %d, %d, %d] %s: %.1fx the bound' % (
                    self.norm, Fr, H, W, C, ('sum', 'sum of squares')[k], ratio))


@pytest.fixture
def audit(monkeypatch):
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import Engine
    rec = Audit()
    apply_stats, ab, gn, decoder_out = ops.groupnorm_apply_stats, ops.groupnorm_ab, Engine._gn, Engine.decoder_out

    def apply_checked(x, gamma, beta, out, stats, chunks_per_frame, *a, **k):
        rec.check(x, stats, chunks_per_frame)
        return apply_stats(x, gamma, beta, out, stats, chunks_per_frame, *a, **k)

    def ab_checked(x, gamma, beta, out, stats=None, chunks_per_frame=0, *a, **k):
        if stats is not None:
            rec.check(x, stats, chunks_per_frame)
        return ab(x, gamma, beta, out, stats, chunks_per_frame, *a, **k)

    def gn_named(self, x, p, *a, **k):
        rec.norm = p
        return gn(self, x, p, *a, **k)

    def decoder_out_named(self, h, norm='decoder.norm_out', *a, **k):
        rec.norm = norm
        return decoder_out(self, h, norm, *a, **k)

    monkeypatch.setattr(ops, 'groupnorm_apply_stats', apply_checked)
    monkeypatch.setattr(ops, 'groupnorm_ab', ab_checked)
    monkeypatch.setattr(Engine, '_gn', gn_named)
    monkeypatch.setattr(Engine, 'decoder_out', decoder_out_named)
    return rec


_models = {}


def _model(name, network_g):
    """One instance per registered model (synthetic weights), built on first use."""
    if name not in _models:
        from pgtformer_b200.registry import ARCH_REGISTRY
        import archs  # noqa: F401
        if name in ('pgtformer', 'tdcrqvae3', 'tdrqvae'):
            g = dict(network_g)
            g['type'] = {'pgtformer': 'PGTFormer', 'tdcrqvae3': 'TDCRQVAE3', 'tdrqvae': 'TDRQVAE'}[name]
        elif name == 'tdcrqvae3_r2':                     # two res blocks per level
            g = copy.deepcopy(network_g)
            g['type'] = 'TDCRQVAE3'
            g['ddconfig']['num_res_blocks'] = 2
        elif name.startswith('rqvae_'):
            from oracle.make_rqvae_golden import CONFIGS
            g = copy.deepcopy(CONFIGS[name[len('rqvae_'):]])
        else:
            g = {'type': {'vqgan': 'VQAutoEncoder', 'codeformer': 'CodeFormer'}[name]}
        kind = g.pop('type')
        _models[name] = ARCH_REGISTRY.get(kind)(**g).to(DEV).eval()
    return _models[name]


def _images(n, H, W, seed):
    return torch.rand(n, 3, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _run(name, m, H, W):
    """The calls of `name` at frame size H x W: every method whose encoder or decoder consumes fused statistics."""
    if name == 'pgtformer':
        m(_images(3, H, W, 1), w=1, adain=True)
    elif name == 'video':
        from pgtformer_b200.video import VideoRestorer
        frames = np.random.RandomState(2).randint(0, 256, size=(5, H, W, 3), dtype=np.uint8)
        out = VideoRestorer(m, w=1.0, adain=True, clips_per_batch=4).restore(frames)
        assert out.shape == frames.shape
    elif name in ('tdcrqvae3', 'tdcrqvae3_r2'):
        _, _, code = m(_images(3, H, W, 3))
        m.decode_code(code)
    elif name == 'tdrqvae':
        x = torch.rand(1, 3, 3, H, W, generator=torch.Generator().manual_seed(4)).to(DEV)
        _, _, code = m(x)
        m.decode_code(code.view(-1, *code.shape[2:]))
    elif name == 'rqvae_r2':
        m(_images(2, H, W, 5))
        z = torch.randn(2, H // 8, W // 8, m.arch.embed_dim, generator=torch.Generator().manual_seed(6))
        m.decode(z.to(DEV))
    elif name == 'rqvae_r1':
        m(_images(1, H, W, 7))
    elif name == 'vqgan':
        m(_images(2, H, W, 8))
    elif name == 'codeformer':
        m(_images(1, H, W, 9), w=0.5, adain=True)
    else:
        raise AssertionError(name)


# (model, H, W) -> the number of fused statistics its calls consume where every level's tile grid divides the frame
# (these counts are unchanged by the rule that fuses statistics only on such grids), or None at sizes some level's grid
# does not divide, where the engines normalise those levels from the tensor and at least one fused statistic remains
CASES = {
    ('pgtformer', 64, 64): 20, ('pgtformer', 64, 192): None, ('pgtformer', 192, 192): None,
    ('video', 64, 192): None,
    ('tdcrqvae3', 64, 64): 30, ('tdcrqvae3', 64, 192): None, ('tdcrqvae3_r2', 64, 64): 48,
    ('tdrqvae', 64, 64): 35, ('tdrqvae', 64, 192): None,
    ('rqvae_r2', 128, 128): 90, ('rqvae_r2', 128, 192): None,
    ('rqvae_r1', 128, 128): 40, ('rqvae_r1', 128, 384): None,
    ('vqgan', 128, 128): 32, ('vqgan', 256, 384): None,
    ('codeformer', 512, 512): 68,
}


@pytest.mark.parametrize('name,H,W', list(CASES))
def test_fused_statistics_match_the_normalised_tensor(network_g, audit, name, H, W):
    m = _model('pgtformer' if name == 'video' else name, network_g)
    _run(name, m, H, W)
    torch.cuda.synchronize()
    print('%s %d x %d: %d fused statistics consumed, %d violations' % (name, H, W, audit.fused, len(audit.violations)))
    assert not audit.violations, '\n'.join(audit.violations)
    assert audit.fused > 0
    if CASES[(name, H, W)] is not None:
        assert audit.fused == CASES[(name, H, W)]


def test_tile_rule_matches_the_launched_grid(tmp_path):
    """conv_tiles_per_frame / conv_tiles_exact mirror the tile choice of conv_impl (gemm_tc.cu), and every statistics
    buffer is sized by them: over frames of 8..256 x 8..256 (multiples of 8) and 64..512 output channels, the 3x3 conv
    (stride 1, and stride 2 as the Downsample runs it) and the upsample conv are launched under the profiler, and the
    tile grid in each launch's description must be the one the two functions describe.  Generic launches carry
    t{frames}x{rows}x{columns}; `halo3` launches use 16-row x 8-column tiles."""
    import csv
    import os
    import re
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_conv, _pack_up2x
    sizes = range(8, 257, 8)
    x = torch.zeros(256 * 256 * 64, dtype=torch.bfloat16, device=DEV)
    out = torch.empty(512 * 512 * 512, dtype=torch.bfloat16, device=DEV)
    path = os.path.join(str(tmp_path), 'launches.csv')
    checked = 0
    for cout in (64, 128, 256, 512):
        w3 = _pack_conv(torch.zeros(cout, 64, 3, 3, device=DEV))
        w4 = _pack_up2x(torch.zeros(cout, 64, 3, 3, device=DEV))
        for mode in ('s1', 's2', 'up2x'):
            expect = []
            ops.profile_begin()
            for H in sizes:
                for W in sizes:
                    xi = x[:H * W * 64].view(1, H, W, 64)
                    if mode == 'up2x':
                        ops.conv_up2x(xi, w4, cout, out[:4 * H * W * cout].view(1, 2 * H, 2 * W, cout))
                        args, n = (H, W, cout, 2, 1, 1), 4
                    else:
                        s = 1 if mode == 's1' else 2
                        ops.conv(xi, w3, cout, out[:H * W // (s * s) * cout].view(1, H // s, W // s, cout), stride=s,
                                 pad_lo=2 - s)
                        args, n = (H, W, cout, 3, s, 2 - s), 1
                    expect += [(args, ops.conv_tiles_per_frame(*args), ops.conv_tiles_exact(*args))] * n
            ops.profile_end(path)
            descs = [r['desc'] for r in csv.DictReader(open(path)) if r['class'] == '0']
            assert len(descs) == len(expect), (cout, mode, len(descs), len(expect))
            for d, (args, tpf, exact) in zip(descs, expect):
                Ho, Wo = (int(v) for v in re.search(r' H(\d+) W(\d+) ', d).groups())
                if d.startswith('halo3 '):
                    tn, th, tw = 1, 16, 8
                else:
                    tn, th, tw = (int(v) for v in re.search(r' t(\d+)x(\d+)x(\d+) ', d).groups())
                grid = -(-Ho // th) * -(-Wo // tw)
                want = grid if tn == 1 else 0
                assert tpf == want, (args, d, tpf)
                assert exact == (want if Ho % th == 0 and Wo % tw == 0 else 0), (args, d, exact)
                checked += 1
    print('%d launches checked' % checked)
