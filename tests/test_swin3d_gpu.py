"""Video-Swin BasicLayer on the H100 kernels (SURVEY 8(f) #4) through the C ABI: the generic 3-D window attention core
vs the oracle restatement of `modules/swin.py` (padding, 3-D shift, clipped windows), and the whole drop-in layer vs the
fixtures minted from the reference's own module."""
import pytest
import torch

from conftest import load_golden
from oracle import swin3d_oracle as S

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def rnd(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.mark.parametrize('B,D,H,W,C,heads,window,shift', [
    (1, 3, 16, 16, 256, 8, (5, 5, 5), (2, 2, 2)),      # D < window: clipped to (3,5,5), N = 75, H/W padded 16 -> 20
    (2, 7, 10, 10, 256, 8, (5, 5, 5), (2, 2, 2)),      # D padded 7 -> 10, shift in all three dims
    (1, 3, 16, 16, 256, 8, (5, 5, 5), (0, 0, 0)),      # unshifted block of the same layer
    (1, 4, 8, 8, 128, 8, (2, 4, 4), (1, 2, 2)),        # no padding, head dim 16
    (1, 2, 12, 8, 512, 8, (2, 4, 4), (1, 2, 2)),       # head dim 64
])
@pytest.mark.parametrize('qkv_bias', [False, True])
def test_window3d_attention_core(B, D, H, W, C, heads, window, shift, qkv_bias):
    """Core only: the qkv rows (and the projection of a zero token for padded positions) are given; compared with the
    oracle's pad / roll / partition / attention / reverse / crop on the same bf16 values.  P is a bf16 MMA operand
    (4e-3 * max|ref| on top of one ulp of the bf16 output)."""
    from pgtformer_b200 import ops
    T = B * D * H * W
    qkv = rnd((T, 3 * C), 1).bfloat16()
    pad = rnd((3 * C,), 2).bfloat16() if qkv_bias else None
    ws, ss = S.window_size_for((D, H, W), window, shift)
    N = ws[0] * ws[1] * ws[2]
    table = 0.5 * rnd(((2 * window[0] - 1) * (2 * window[1] - 1) * (2 * window[2] - 1), heads), 3)
    index = S.relative_position_index(window)
    bias = table[index[:N, :N].reshape(-1)].view(N, N, heads).permute(2, 0, 1).contiguous()
    out = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    ops.window3d_attention(qkv.to(DEV), B, D, H, W, C, heads, window, shift, bias.to(DEV), out,
                           pad_qkv=pad.to(DEV) if pad is not None else None)
    torch.cuda.synchronize()
    # oracle on the projected rows: pad with the zero-token projection, then exactly swin3d_oracle.block's geometry
    x = qkv.float().view(B, D, H, W, 3 * C)
    pd, pb, pr = (ws[0] - D % ws[0]) % ws[0], (ws[1] - H % ws[1]) % ws[1], (ws[2] - W % ws[2]) % ws[2]
    xp = torch.nn.functional.pad(x, (0, 0, 0, pr, 0, pb, 0, pd))
    if pad is not None:
        m = torch.zeros(B, D + pd, H + pb, W + pr, 1)
        m[:, :D, :H, :W] = 1
        xp = xp * m + pad.float().view(1, 1, 1, 1, -1) * (1 - m)
    Dp, Hp, Wp = xp.shape[1:4]
    shifted = any(s > 0 for s in ss)
    if shifted:
        xp = torch.roll(xp, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    xw = S.partition(xp, ws)
    d = C // heads
    q = xw[..., :C].reshape(-1, N, heads, d).permute(0, 2, 1, 3) * d ** -0.5
    k = xw[..., C:2 * C].reshape(-1, N, heads, d).permute(0, 2, 1, 3)
    v = xw[..., 2 * C:].reshape(-1, N, heads, d).permute(0, 2, 1, 3)
    attn = q @ k.transpose(-2, -1) + bias[None]
    if shifted:
        mask = S.shift_mask(Dp, Hp, Wp, ws, ss)
        attn = (attn.view(-1, mask.shape[0], heads, N, N) + mask[None, :, None]).view(-1, heads, N, N)
    ow = (attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, N, C)
    ref = S.reverse(ow, ws, B, Dp, Hp, Wp)
    if shifted:
        ref = torch.roll(ref, shifts=ss, dims=(1, 2, 3))
    ref = ref[:, :D, :H, :W].reshape(T, C)
    got = out.float().cpu()
    assert torch.isfinite(got).all(), 'unwritten rows'
    err = (got - ref).abs()
    tol = ref.abs() * 2.0 ** -8 + 4e-3 * ref.abs().max()
    assert not (err > tol).any(), 'max err %.3e (max|ref| %.3e)' % (err.max(), ref.abs().max())


@pytest.mark.parametrize('case', ['a', 'b'])
def test_basic_layer_against_reference_golden(case):
    """The drop-in `modules.swin.BasicLayer` with the stand-in checkpoint vs the output of the reference's own module
    (depth x (2 LayerNorms, 4 bf16 GEMMs, attention) of bf16 activations: 2e-2 * max|ref|)."""
    from modules.swin import BasicLayer
    c = S.SWIN_CASES[case]
    layer = BasicLayer(c['dim'], c['depth'], c['heads'], c['window'])
    layer.load_state_dict(S.synth_state(layer.state_dict(), c['seed']), strict=True)
    layer = layer.to(DEV)
    g = load_golden('swin3d_%s.pt' % case)
    y = layer(S.case_input(case).to(DEV))
    assert y.shape == g['out'].shape and y.dtype == torch.float32
    err = (y.cpu() - g['out'].float()).abs().max().item()
    print('swin3d %s: max err %.3e of max|ref| %.3f' % (case, err, g['out_absmax']))
    assert err < 2e-2 * g['out_absmax']
