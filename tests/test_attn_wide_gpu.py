"""The wide-head attention core (attn_wide_tc.cu: `pgt_mha_fwd` with d = 256 / 512, the dense AttnBlock core of TDRQVAE)
against an fp64 softmax(q k^T d^-1/2) v on the same bf16 inputs, within 4e-3 * max|ref| (the flash-kernel bound: the
probabilities P are bf16 operands of the P V product), plus the properties the kernel must keep: no reads across frames,
strided q / k / v views, degenerate and very large scores, the d = 64 path unchanged, and both bindings."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ops():
    from pgtformer_b200 import ops as o
    return o


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def ref_attn(q, k, v, clips, L, heads, d, chunk=2048):
    """fp64 softmax(q k^T / sqrt(d)) v per (clip, head) on the bf16 values; q / k / v row views [clips*L, >= heads*d]."""
    out = torch.empty(clips * L, heads * d, dtype=torch.float64, device=DEV)
    for c in range(clips):
        for h in range(heads):
            rows, cols = slice(c * L, (c + 1) * L), slice(h * d, (h + 1) * d)
            K, V = k[rows, cols].double(), v[rows, cols].double()
            for i in range(0, L, chunk):
                Q = q[c * L + i:c * L + min(i + chunk, L), cols].double()
                out[c * L + i:c * L + min(i + chunk, L), cols] = torch.softmax(Q @ K.t() / math.sqrt(d), -1) @ V
    return out


def check(got, ref, what, rel=4e-3):
    got = got.double()
    assert torch.isfinite(got).all(), what + ': non-finite output'
    mx = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= rel * mx, '%s: max err %.3e > %.0e * max|ref| %.3e' % (what, err, rel, mx)


def run(q, k, v, clips, L, heads, d, out=None):
    if out is None:
        out = torch.empty(clips * L, heads * d, dtype=torch.bfloat16, device=DEV)
    ops().mha(q, k, v, clips, L, heads, d, out)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('d', [256, 512])
@pytest.mark.parametrize('L', [16, 80, 100, 1024, 4096, 16384])
def test_wide_mha_vs_fp64(d, L):
    clips = 1 if L == 16384 else 3
    T = clips * L
    q, k, v = rnd((T, d), 1000 + L, 2.0), rnd((T, d), 2000 + L), rnd((T, d), 3000 + L)
    out = run(q, k, v, clips, L, 1, d)
    check(out, ref_attn(q, k, v, clips, L, 1, d), 'd=%d L=%d' % (d, L))


@pytest.mark.parametrize('d', [256, 512])
def test_wide_mha_two_heads(d):
    clips, L, heads = 2, 208, 2
    q, k, v = (rnd((clips * L, heads * d), 40 + i, 1.5) for i in range(3))
    check(run(q, k, v, clips, L, heads, d), ref_attn(q, k, v, clips, L, heads, d), 'two heads d=%d' % d)


@pytest.mark.parametrize('d', [256, 512])
def test_wide_mha_strided_views(d):
    """q, k, v as column slices of one [F*L, 3C] projection output (how AttnBlock calls it), out a slice of a wider
    buffer whose other columns must stay untouched."""
    clips, L = 2, 272
    qkv = rnd((clips * L, 3 * d), 50, 1.5)
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    buf = torch.full((clips * L, 2 * d), float('nan'), dtype=torch.bfloat16, device=DEV)
    run(q, k, v, clips, L, 1, d, out=buf[:, d:])
    check(buf[:, d:], ref_attn(q, k, v, clips, L, 1, d), 'strided d=%d' % d)
    assert torch.isnan(buf[:, :d].float()).all()


@pytest.mark.parametrize('d', [256, 512])
@pytest.mark.parametrize('L', [16, 80, 1040])
def test_wide_mha_no_cross_frame_reads(d, L):
    """A neighbouring frame of huge values leaves the other frames' outputs bit for bit unchanged: key tiles running past
    L are masked by key index, not by TMA zero fill."""
    clips = 3
    q, k, v = (rnd((clips * L, d), 60 + i, 1.5) for i in range(3))
    base = run(q, k, v, clips, L, 1, d)
    q2, k2, v2 = q.clone(), k.clone(), v.clone()
    for t in (q2, k2, v2):
        t[L:2 * L] = 3.0e4
    other = run(q2, k2, v2, clips, L, 1, d)
    assert torch.equal(base[:L], other[:L]) and torch.equal(base[2 * L:], other[2 * L:])
    check(base, ref_attn(q, k, v, clips, L, 1, d), 'd=%d L=%d' % (d, L))


@pytest.mark.parametrize('d', [256, 512])
def test_wide_mha_equal_scores_give_mean_of_v(d):
    clips, L = 2, 4096
    q = torch.zeros(clips * L, d, dtype=torch.bfloat16, device=DEV)
    k, v = rnd((clips * L, d), 70), rnd((clips * L, d), 71)
    out = run(q, k, v, clips, L, 1, d)
    ref = v.double().view(clips, L, d).mean(1, keepdim=True).expand(clips, L, d).reshape(clips * L, d)
    check(out, ref, 'equal scores d=%d' % d)


@pytest.mark.parametrize('d', [256, 512])
def test_wide_mha_large_scores(d):
    """Scores of magnitude ~1e3 after the d^-1/2 scale: every key tile raises the reference exponent far beyond the
    first tile's, which must neither overflow p nor lose the row."""
    clips, L = 1, 1024
    q, k, v = rnd((L, d), 80, 18.0), rnd((L, d), 81, 18.0), rnd((L, d), 82)
    s = (q.double() @ k.double().t()) / math.sqrt(d)
    assert s.abs().max().item() > 1e3
    check(run(q, k, v, clips, L, 1, d), ref_attn(q, k, v, clips, L, 1, d), 'large scores d=%d' % d)


def test_d64_unchanged():
    """d = 64 (the global transformer's heads) still runs the mha_tc / mma.sync kernels: outputs bit-identical to the
    library before the wide-head kernel was added, recorded on the same inputs."""
    g = torch.load(os.path.join(ROOT, 'tests', 'golden', 'mha_d64_outputs.pt'), map_location='cpu')
    for case in g['cases']:
        clips, L, heads, seed = case['clips'], case['L'], case['heads'], case['seed']
        q, k, v = (rnd((clips * L, heads * 64), seed + i) for i in range(3))
        out = run(q, k, v, clips, L, heads, 64)
        assert torch.equal(out.cpu(), case['out']), case


@pytest.mark.parametrize('d', [256, 512])
def test_wide_mha_torch_op_equals_ctypes(d):
    from pgtformer_b200 import torch_ops
    t = torch_ops.load()
    clips, L = 2, 336
    q, k, v = (rnd((clips * L, d), 90 + i, 1.5) for i in range(3))
    m1 = run(q, k, v, clips, L, 1, d)
    m2 = torch.empty_like(m1)
    t.mha_fwd(q, k, v, clips, L, 1, d, m2)
    torch.cuda.synchronize()
    assert torch.equal(m1, m2)


def test_unsupported_width_raises():
    q = torch.zeros(64, 128, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(Exception):
        ops().mha(q, q, q, 1, 64, 1, 128, torch.empty_like(q))
