"""GPU tests at frames with H != W, where one 64-pixel side leaves level 4 and the mid layers one window row (or column)
deep.  The reference's get_window_size (`modules/rstt_layers.py:90-114`) then drops the shift of that axis only: the
other axis is still rolled and masked.  Checked here: both window-attention kernels against an fp64 evaluation of that
rule, the engine's Swin layers and parsing branch against the oracle, and PGTFormer and the TDCRQVAE3 codec against
the reference's own outputs (oracle/make_golden.py --nonsquare, oracle/make_codec_golden.py).  Bounds are those of the
square tests: tests/test_numeric_range_gpu.py, tests/test_tc_kernels_gpu.py and tests/test_model_gpu.py."""
import pytest
import torch

from conftest import golden_sample, load_golden
from oracle.make_golden import NONSQUARE_CASES, golden_input, nonsquare_name
from test_model_gpu import bf_sd, eng, model, nhwc, psnr, rand_fm, relerr, sampled_relerr  # noqa: F401 (fixtures)
from test_numeric_range_gpu import check_close, window2d_bias, window2d_reference, window_qkv

pytestmark = pytest.mark.gpu
DEV = 'cuda'

# (C, H, W, clips): a single window row or column with 2-5 windows along the other axis; 4 x 4 is the square control
WINDOW_SHAPES = [(512, 4, 12, 1), (512, 12, 4, 2), (256, 4, 8, 3), (256, 8, 4, 1), (512, 4, 20, 1), (512, 4, 4, 1)]
WINDOW_IDS = ['C%d-%dx%d-c%d' % s for s in WINDOW_SHAPES]


def window_inputs(C, H, W, clips, scores, seed):
    """qkv bf16 [T, 3C] and the expanded bias [8, 48, 48]: N(0, 1) inputs with a 0.5-std table ('normal'), or the
    large-score inputs of test_numeric_range_gpu.py, where the -100 shift mask no longer zeroes a masked key."""
    from pgtformer_b200.weights import relative_position_index
    T = clips * 3 * H * W
    if scores == 'large':
        return window_qkv(T, C, seed), window2d_bias(8, seed + 1)
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(T, 3 * C, generator=g).bfloat16()
    table = 0.5 * torch.randn(245, 8, generator=g)
    return qkv, table[relative_position_index().view(-1)].view(48, 48, 8).permute(2, 0, 1).contiguous()


def run_window(kernel, qkv, clips, H, W, C, shift, bias_tab):
    from pgtformer_b200 import ops
    out = torch.full((qkv.shape[0], C), float('nan'), dtype=torch.bfloat16, device=DEV)
    if kernel == 'mma_sync':
        ops.window_attention(qkv, clips, H, W, C, 8, shift, bias_tab, out)
    else:
        assert ops.window_attention_tc(qkv, clips, H, W, C, 8, shift, ops.window_tables(bias_tab), out) is not None
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('C,H,W,clips', WINDOW_SHAPES, ids=WINDOW_IDS)
@pytest.mark.parametrize('shifted', [False, True])
@pytest.mark.parametrize('scores', ['normal', 'large'])
@pytest.mark.parametrize('kernel', ['tc', 'mma_sync'])
def test_window_attention_per_axis_shift(C, H, W, clips, shifted, scores, kernel):
    qkv, bias_tab = window_inputs(C, H, W, clips, scores, 900 + C + H)
    qd, bd = qkv.to(DEV), bias_tab.to(DEV)
    out = run_window(kernel, qd, clips, H, W, C, 2 if shifted else 0, bd)
    ref = window2d_reference(qd, clips, H, W, C, 8, bd, shifted)
    check_close(out, ref, '%s %s %dx%d shifted=%s' % (kernel, scores, H, W, shifted), rel=4e-3)


@pytest.mark.parametrize('C,H,W,clips', WINDOW_SHAPES, ids=WINDOW_IDS)
def test_window_attention_tc_matches_mma_sync_nonsquare(C, H, W, clips):
    """As test_window_attention_tc_matches_mma_sync_kernel: the two kernels agree to bf16 rounding."""
    qkv, bias_tab = window_inputs(C, H, W, clips, 'normal', 950 + C + H)
    qd, bd = qkv.to(DEV), bias_tab.to(DEV)
    for shift in (0, 2):
        a = run_window('mma_sync', qd, clips, H, W, C, shift, bd).float()
        b = run_window('tc', qd, clips, H, W, C, shift, bd).float()
        d = (a - b).abs().max().item()
        assert d <= 4e-3 * a.abs().max().item() + 2.0 ** -7, (shift, d)


@pytest.mark.parametrize('prefix,H,W,clips', [('encoder.down.4.attn.0', 4, 12, 1), ('decoder.mid.attn_1', 12, 4, 2),
                                              ('encoder.mid.attn_1', 4, 8, 1)])
def test_encoder_layer_nonsquare(eng, bf_sd, prefix, H, W, clips):
    from oracle import pgt_oracle as O
    x = rand_fm((3 * clips, H, W, 512), 12)
    got = eng.encoder_layer(x.to(DEV), prefix, 8, 2)
    ref = nhwc(O.encoder_layer(bf_sd, prefix, x.float().permute(0, 3, 1, 2), 8, 2))
    assert relerr(got, ref) < 1.5e-2


@pytest.mark.parametrize('H,W', [(64, 192), (192, 64)])
def test_parsing_net_and_pos_nonsquare(eng, bf_sd, H, W):
    """BiSeNet's heads are resized to (H/16, W/16) with x and y scaled apart (align_corners bilinear)."""
    from oracle import pgt_oracle as O
    x = torch.rand(3, 3, H, W, generator=torch.Generator().manual_seed(13))
    got = eng.parse_pos(x.to(DEV))
    mean = torch.tensor(O.IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(O.IMAGENET_STD).view(1, 3, 1, 1)
    ref = nhwc(O.conv(bf_sd, 'convpos', O.bisenet(bf_sd, 'conditionnet', (x - mean) / std)))
    assert relerr(got.view(ref.shape), ref) < 3e-2      # bound of test_parsing_net_and_pos


@pytest.mark.parametrize('fixture', [nonsquare_name(*c) for c in NONSQUARE_CASES])
def test_forward_against_reference_golden_nonsquare(model, fixture):
    """The bounds of test_forward_against_reference_golden, and the L2-argmin codes of TDCRQVAE3.forward as in
    test_vq_path_codes_against_reference_golden."""
    g = load_golden(fixture)
    x = golden_input(g['seed'], g['b'], g['H'], g['W']).to(DEV)
    out, logits, lq = model(x, w=1, adain=True)
    assert sampled_relerr(lq, g, 'lq_feat') < 2.5e-2
    assert sampled_relerr(logits, g, 'logits') < 2.5e-2
    agree = (logits.argmax(-1).cpu() == g['codes']).float().mean().item()
    print('code agreement vs reference: %.4f' % agree)
    assert agree > 0.90
    out_tf, _, _ = model(x, w=1, adain=True, force_codes=g['codes'])
    p = psnr(golden_sample(out_tf, g, 'out'), g['out'])
    print('teacher-forced PSNR vs reference out: %.2f dB' % p)
    assert p > 35.0 and sampled_relerr(out_tf, g, 'out') < 8e-2
    _, _, codes = model.forward_vq(x, code_only=True)
    assert codes.shape == g['vq_codes'].shape
    assert (codes.cpu() == g['vq_codes']).float().mean().item() > 0.9


def test_codec_against_reference_golden_nonsquare(model):
    """encode and decode_code at 64 x 192 with the bounds of test_encode_decode_against_reference_golden_128_b2."""
    g = load_golden('tdcrqvae3_codec_b1_64x192_seed23.pt')
    x = golden_input(g['seed'], g['b'], g['H'], g['W']).to(DEV)
    z_e = model.encode(x)
    assert sampled_relerr(z_e, g, 'z_e') < 2.5e-2
    for key, code in (('out', g['codes']), ('out_code', g['code'])):
        out = model.decode_code(code.to(DEV))
        assert psnr(golden_sample(out, g, key), g[key]) > 35.0 and sampled_relerr(out, g, key) < 8e-2, key
