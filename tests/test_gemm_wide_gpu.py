"""The 128 x 256 wgmma tiles (gemm_tc_kernel<256>) that dispatch_gemm picks for N > 128 when the shape has enough tiles
to fill the GPU.  Each case is large enough to take that path (asserted from the launch descriptions), and checks
  * convs against an fp64 reference on the bf16-rounded operands: 1e-3 * max|ref| for fp32 outputs, one bf16 ulp (+ that
    floor) for bf16 outputs, 6e-3 for the upsample conv (its tap-summed phase weights are rounded to bf16 once more);
  * bit equality with the same product launched as 128-column slices (the 128-wide kernel): every output element
    accumulates its k-blocks in the same order in both kernels.  A stride-1 3x3 conv with Cout <= 128 runs on the halo
    kernel instead, whose k order (channel block, then tap) matches only for Cin <= 64, so only those are compared."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def ops():
    from pgtformer_b200 import ops as o
    return o


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def bf(x):
    return x.to(torch.bfloat16)


def check_close(got, ref, what, bf16_out=False, rel=1e-3):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), what + ': non-finite output'
    mx = ref.abs().max().item()
    err = (got - ref).abs()
    tol = (ref.abs() * 2.0 ** -8 if bf16_out else 0) + rel * mx
    bad = err > tol
    assert not bad.any(), '%s: %d elements out of tolerance (max err %.3e, max|ref| %.3e)' % (
        what, int(bad.sum()), err.max().item(), mx)


def launches(fn, tmp_path):
    """Runs fn under the library's launch profiler -> descriptions of the GEMM-class launches."""
    o = ops()
    path = os.path.join(str(tmp_path), 'launches.csv')
    o.profile_begin()
    fn()
    o.profile_end(path)
    import csv
    return [r['desc'] for r in csv.DictReader(open(path)) if r['class'] == '0']


def assert_wide(descs):
    assert descs and all(' BN256 ' in d for d in descs), descs


def pack_conv_weight(w):
    co, ci, kh, kw = w.shape
    cp = (ci + 63) // 64 * 64
    wp = torch.zeros(co, kh * kw, cp, device=w.device)
    wp[:, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return bf(wp.reshape(co, kh * kw * cp)).contiguous()


def conv_ref(x, w, b, stride=1, pad=(1, 1, 1, 1)):
    y = F.conv2d(F.pad(x.double().permute(0, 3, 1, 2), pad), w.double(), None if b is None else b.double(), stride=stride)
    return y.permute(0, 2, 3, 1)


def sliced(run, N, step=128):
    """run(n0, n1) launches the product for output columns [n0, n1)."""
    for n0 in range(0, N, step):
        run(n0, min(N, n0 + step))


# ------------------------------------------------------------------------------------ convs
@pytest.mark.parametrize('Cin,Cout,out_dt', [(64, 256, torch.float32), (128, 512, torch.bfloat16),
                                             (64, 448, torch.float32), (64, 256, torch.bfloat16), (96, 256, torch.bfloat16)])
def test_conv3x3_wide(Cin, Cout, out_dt, tmp_path):
    """Cout 448: ragged second tile; Cin 96: channel tail zero-filled by TMA; 80 x 80: ragged 64-pixel-wide tiles."""
    o = ops()
    Fr, H, W = 3, 80, 80
    x = bf(rnd((Fr, H, W, Cin), 1))
    w = bf(rnd((Cout, Cin, 3, 3), 2, (9 * Cin) ** -0.5)).float()
    b = rnd((Cout,), 3, 0.1)
    wp = pack_conv_weight(w)
    out = torch.empty(Fr, H, W, Cout, dtype=out_dt, device=DEV)
    assert_wide(launches(lambda: o.conv(x, wp, Cout, out, bias=b, act=o.ACT_SILU), tmp_path))
    check_close(out, F.silu(conv_ref(x, w, b)), 'conv3x3 wide', bf16_out=out_dt == torch.bfloat16)
    if Cin > 64:
        return
    ref128 = torch.empty_like(out)
    sliced(lambda n0, n1: o.conv(x, wp[n0:n1], n1 - n0, ref128[..., n0:n1], bias=b[n0:n1], act=o.ACT_SILU), Cout)
    assert torch.equal(out, ref128)


@pytest.mark.parametrize('pad_lo', [0, 1])
def test_conv3x3_stride2_wide(pad_lo, tmp_path):
    o = ops()
    Fr, H, W, Cin, Cout = 3, 160, 160, 128, 256
    x = bf(rnd((Fr, H, W, Cin), 10))
    w = bf(rnd((Cout, Cin, 3, 3), 11, (9 * Cin) ** -0.5)).float()
    b = rnd((Cout,), 12, 0.1)
    wp = pack_conv_weight(w)
    out = torch.empty(Fr, H // 2, W // 2, Cout, dtype=torch.float32, device=DEV)
    assert_wide(launches(lambda: o.conv(x, wp, Cout, out, stride=2, pad_lo=pad_lo, bias=b), tmp_path))
    pad = (0, 1, 0, 1) if pad_lo == 0 else (1, 1, 1, 1)
    check_close(out, conv_ref(x, w, b, stride=2, pad=pad), 'conv s2 wide')
    ref128 = torch.empty_like(out)
    sliced(lambda n0, n1: o.conv(x, wp[n0:n1], n1 - n0, ref128[..., n0:n1], stride=2, pad_lo=pad_lo, bias=b[n0:n1]), Cout)
    assert torch.equal(out, ref128)


@pytest.mark.parametrize('res_dt,out_dt', [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32),
                                           (torch.float32, torch.bfloat16)])
def test_conv_residual_wide(res_dt, out_dt, tmp_path):
    """Residual TMA-loaded into the 2-slot staging ring (same dtype), or read per thread (mixed dtypes); plus the
    ReLU-after-residual of a ResNet block."""
    o = ops()
    Fr, H, W, C = 3, 80, 80, 256
    x = bf(rnd((Fr, H, W, C), 20))
    w = bf(rnd((C, C, 3, 3), 21, (9 * C) ** -0.5)).float()
    b = rnd((C,), 22, 0.1)
    res = rnd((Fr, H, W, C), 23).to(res_dt)
    wp = pack_conv_weight(w)
    y = conv_ref(x, w, b)
    out = torch.empty(Fr, H, W, C, dtype=out_dt, device=DEV)
    assert_wide(launches(lambda: o.conv(x, wp, C, out, bias=b, residual=res), tmp_path))
    check_close(out, y + res.double(), 'conv+residual wide', bf16_out=out_dt == torch.bfloat16)
    o.conv(x, wp, C, out, bias=b, act=o.ACT_RELU, residual=res, relu_after_res=True)
    check_close(out, F.relu(y + res.double()), 'conv relu-after-residual wide', bf16_out=out_dt == torch.bfloat16)


def test_conv_nchw_and_channel_slice_wide(tmp_path):
    """fp32 NCHW output (per-thread stores) and a bf16 output written into a channel slice of a wider buffer."""
    o = ops()
    Fr, H, W, Cin, Cout = 3, 80, 80, 64, 256
    x = bf(rnd((Fr, H, W, Cin), 30))
    w = bf(rnd((Cout, Cin, 3, 3), 31, (9 * Cin) ** -0.5)).float()
    b = rnd((Cout,), 32, 0.1)
    wp = pack_conv_weight(w)
    y = conv_ref(x, w, b)
    nchw = torch.empty(Fr, Cout, H, W, dtype=torch.float32, device=DEV)
    assert_wide(launches(lambda: o.conv(x, wp, Cout, nchw, bias=b, nchw=True), tmp_path))
    check_close(nchw, y.permute(0, 3, 1, 2), 'conv nchw wide')
    buf = torch.zeros(Fr, H, W, Cout + 192, dtype=torch.bfloat16, device=DEV)
    assert_wide(launches(lambda: o.conv(x, wp, Cout, buf[..., 64:64 + Cout], bias=b), tmp_path))
    check_close(buf[..., 64:64 + Cout], y, 'conv channel slice wide', bf16_out=True)
    assert buf[..., :64].abs().max() == 0 and buf[..., 64 + Cout:].abs().max() == 0


def test_conv_groupnorm_stats_wide(tmp_path):
    """Fused GroupNorm statistics with 16 channels per group (Cout 512) from 256-wide tiles."""
    o = ops()
    Fr, H, W, Cin, C = 3, 64, 64, 128, 512
    x = bf(rnd((Fr, H, W, Cin), 40))
    w = bf(rnd((C, Cin, 3, 3), 41, (9 * Cin) ** -0.5)).float()
    b = rnd((C,), 42, 0.1)
    gam, bet = 1 + 0.1 * rnd((C,), 43), 0.1 * rnd((C,), 44)
    tpf = o.conv_tiles_per_frame(H, W, C)
    assert tpf > 0
    stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
    y = torch.empty(Fr, H, W, C, dtype=torch.bfloat16, device=DEV)
    assert_wide(launches(lambda: o.conv(x, pack_conv_weight(w), C, y, bias=b, gn_stats=stats), tmp_path))
    check_close(y, conv_ref(x, w, b), 'producer', bf16_out=True)
    out = torch.empty_like(y)
    o.groupnorm_apply_stats(y, gam, bet, out, stats, tpf * 4)
    gref = F.silu(F.group_norm(y.double().permute(0, 3, 1, 2), 32, gam.double(), bet.double(), eps=1e-6))
    check_close(out, gref.permute(0, 2, 3, 1), 'fused-stats groupnorm wide', bf16_out=True, rel=3e-3)


def test_conv_up2x_groupnorm_stats_wide(tmp_path):
    """The four upsample phases (strided placement) with fused statistics, 8 channels per group."""
    from pgtformer_b200.engine import _pack_up2x
    o = ops()
    Fr, H, W, C = 6, 64, 64, 256
    x = bf(rnd((Fr, H, W, C), 50))
    w = bf(rnd((C, C, 3, 3), 51, (9 * C) ** -0.5)).float()
    b = rnd((C,), 52, 0.1)
    gam, bet = 1 + 0.1 * rnd((C,), 53), 0.1 * rnd((C,), 54)
    tpf = o.conv_tiles_per_frame(H, W, C, 2, 1, 1)
    assert tpf > 0
    stats = torch.zeros(Fr * 16 * tpf * 64, dtype=torch.float32, device=DEV)
    y = torch.empty(Fr, 2 * H, 2 * W, C, dtype=torch.bfloat16, device=DEV)
    descs = launches(lambda: o.conv_up2x(x, _pack_up2x(w), C, y, bias=b, gn_stats=stats), tmp_path)
    assert len(descs) == 4
    assert_wide(descs)
    up = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode='nearest')
    ref = F.conv2d(up, w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    check_close(y, ref, 'conv up2x wide', bf16_out=True, rel=6e-3)
    out = torch.empty_like(y)
    o.groupnorm_apply_stats(y, gam, bet, out, stats, 16 * tpf)
    gref = F.silu(F.group_norm(y.double().permute(0, 3, 1, 2), 32, gam.double(), bet.double(), eps=1e-6))
    check_close(out, gref.permute(0, 2, 3, 1), 'up2x fused-stats groupnorm wide', bf16_out=True, rel=3e-3)


# ------------------------------------------------------------------------------------ linears
@pytest.mark.parametrize('N', [256, 768, 1000, 1536])
@pytest.mark.parametrize('out_dt,res_dt', [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32),
                                           (torch.float32, None)])
def test_linear_wide_equals_128_slices(N, out_dt, res_dt, tmp_path):
    """M = 17000 (ragged last row tile) and K = 520 (k tail): bit-identical to 128-column launches of the same product."""
    o = ops()
    M, K = 17000, 520
    a = bf(rnd((M, K), 60))
    w = bf(rnd((N, K), 61, K ** -0.5))
    b = rnd((N,), 62, 0.1)
    r = rnd((M, N), 63).to(res_dt) if res_dt is not None else None
    out = torch.empty(M, N, dtype=out_dt, device=DEV)
    assert_wide(launches(lambda: o.linear(a, w, out, bias=b, act=o.ACT_GELU, residual=r), tmp_path))
    ref = F.gelu(a.double() @ w.double().t() + b.double()) + (r.double() if r is not None else 0)
    check_close(out, ref, 'linear wide', bf16_out=out_dt == torch.bfloat16)
    ref128 = torch.empty_like(out)
    sliced(lambda n0, n1: o.linear(a, w[n0:n1], ref128[:, n0:n1], bias=b[n0:n1], act=o.ACT_GELU,
                                   residual=r[:, n0:n1] if r is not None else None), N)
    assert torch.equal(out, ref128)


def test_linear_wide_torch_ops_binding():
    """torch.ops.pgt.linear and the ctypes binding reach the same 256-wide launch: identical bits."""
    from pgtformer_b200 import torch_ops
    o = ops()
    t = torch_ops.load()
    M, N, K = 17000, 768, 512
    a = bf(rnd((M, K), 70))
    w = bf(rnd((N, K), 71, K ** -0.5))
    b = rnd((N,), 72, 0.1)
    r = bf(rnd((M, N), 73))
    y1 = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    y2 = torch.empty_like(y1)
    o.linear(a, w, y1, bias=b, act=o.ACT_GELU, residual=r)
    t.linear(a, w, b, o.ACT_GELU, r, y2)
    assert torch.equal(y1, y2)
