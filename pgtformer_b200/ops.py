"""Tensor-level wrappers over the C ABI (ctypes): validate shapes / strides, pass raw device
pointers and the current CUDA stream.  No computation happens in Python or ATen here.

Activations are channels-last: feature maps are [F, H, W, C] tensors (possibly channel-slice
views of a wider buffer: stride(-1) == 1, stride(-2) == ld), token matrices are [T, C].
"""
import ctypes

import torch

from . import _lib as L
from ._lib import (ACT_GELU, ACT_LRELU02, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SILU, BF16, EPI_PLAIN,  # noqa: F401
                   EPI_SFT, F32, OUT_NCHW, OUT_NHWC, Epilogue)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(t=None):
    """Current CUDA stream of the tensor's device (of the current device when no tensor is given)."""
    if t is not None:
        return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dt(t):
    if t.dtype == torch.bfloat16:
        return BF16
    if t.dtype == torch.float32:
        return F32
    raise TypeError('unsupported dtype %s' % t.dtype)


def _rows(t):
    """Views a channels-last tensor as (rows, C, ld); requires a uniform row stride."""
    assert t.is_cuda and t.stride(-1) == 1, 'expected a CUDA channels-last tensor'
    C = t.shape[-1]
    ld = t.stride(-2) if t.dim() > 1 else C
    rows = 1
    exp = ld
    for d in range(t.dim() - 2, -1, -1):
        assert t.shape[d] == 1 or t.stride(d) == exp, 'non-uniform row stride'
        exp *= t.shape[d]
        rows *= t.shape[d]
    return rows, C, ld


def make_epilogue(out, bias=None, act=ACT_NONE, residual=None, sft_scale=None, sft_w=0.0, nchw=False,
                  relu_after_res=False, gn_stats=None):
    """sft_w: the SFT fusion weight, a number or (convolutions only) a device fp32 tensor of one weight per output
    frame."""
    ep = Epilogue()
    ep.flags = 1 if relu_after_res else 0
    if gn_stats is not None:
        assert gn_stats.dtype == torch.float32 and gn_stats.is_contiguous()
        ep.gn_stats = gn_stats.data_ptr()
    ep.bias = bias.data_ptr() if bias is not None else None
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    ep.act = act
    ep.mode = EPI_SFT if sft_scale is not None else EPI_PLAIN
    if residual is not None:
        _, _, ldr = _rows(residual)
        ep.residual, ep.ldr, ep.res_dtype = residual.data_ptr(), ldr, _dt(residual)
    if sft_scale is not None:
        _, _, lda = _rows(sft_scale)
        assert sft_scale.dtype == torch.bfloat16
        ep.aux, ep.ldaux = sft_scale.data_ptr(), lda
        if torch.is_tensor(sft_w):
            assert sft_w.dtype == torch.float32 and sft_w.is_contiguous() and sft_w.device == out.device
            ep.sft_wf = sft_w.data_ptr()
        else:
            ep.sft_w = float(sft_w)
    ep.out = out.data_ptr()
    ep.out_dtype = _dt(out)
    if nchw:
        assert out.is_contiguous() and out.dtype == torch.float32
        ep.out_layout, ep.ldo = OUT_NCHW, 0
    else:
        ep.out_layout, ep.ldo = OUT_NHWC, _rows(out)[2]
    return ep


def gn_stats_supported(C):
    """Whether a C-channel output can carry fused GroupNorm(32) statistics (the gn_stats argument below): 2, 4, 8, 16
    or 32 channels per group, as setup_epilogue_maps in gemm_tc.cu requires."""
    return C % 32 == 0 and C // 32 in (2, 4, 8, 16, 32)


def linear(a, w, out, bias=None, act=ACT_NONE, residual=None, K=None, N=None, relu_after_res=False, gn_stats=None):
    """out[T,N] = act(a[T,K] @ w[N,K]^T + bias) (+ residual).  a, w bf16; out bf16 / fp32."""
    lib = L.load()
    M, Ka, lda = _rows(a)
    Nw, Kw = w.shape
    K = K if K is not None else min(Ka, Kw)
    N = N if N is not None else Nw
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.stride(1) == 1
    assert _rows(out)[0] == M and out.shape[-1] >= N
    ep = make_epilogue(out, bias, act, residual, relu_after_res=relu_after_res, gn_stats=gn_stats)
    L.check(lib.pgt_linear_bf16(_p(a), lda, _p(w), w.stride(0), M, N, K, ctypes.byref(ep), _stream()))
    return out


def conv(x, wp, cout, out, ksize=3, stride=1, pad_lo=1, bias=None, act=ACT_NONE, residual=None, sft_scale=None,
         sft_w=0.0, nchw=False, relu_after_res=False, gn_stats=None):
    """Implicit-GEMM conv on [F,H,W,Cin] bf16 with packed weights wp [>=cout, k*k*CinPad]; sft_w: a number or a
    device fp32 [F] tensor of per-frame weights."""
    lib = L.load()
    F, H, W, Cin = x.shape
    assert not torch.is_tensor(sft_w) or sft_w.numel() == F
    assert x.dtype == torch.bfloat16 and x.stride(3) == 1 and x.stride(1) == W * x.stride(2) and \
        (F == 1 or x.stride(0) == H * x.stride(1))
    ep = make_epilogue(out, bias, act, residual, sft_scale, sft_w, nchw, relu_after_res, gn_stats)
    L.check(lib.pgt_conv_bf16(_p(x), F, H, W, Cin, x.stride(2), _p(wp), wp.stride(0), cout, ksize, stride, pad_lo,
                              ctypes.byref(ep), _stream()))
    return out


def conv_rgb(x_nchw, wp, bias, out, ksize, stride, pad, act=ACT_NONE, mean3=None, std3=None, gn_stats=None):
    """Cin = 3 conv on the tensor cores straight from the fp32 NCHW image; wp [Cout, Kpad] bf16 (engine._pack_rgb), Cout 64
    (3x3 / 1 and 7x7 / 2) or 128 (3x3 / 1)."""
    lib = L.load()
    F, C, H, W = x_nchw.shape
    assert C == 3 and x_nchw.dtype == torch.float32 and x_nchw.is_contiguous() and wp.dtype == torch.bfloat16
    m = (ctypes.c_float * 3)(*[float(v) for v in mean3]) if mean3 is not None else None
    s = (ctypes.c_float * 3)(*[float(v) for v in std3]) if std3 is not None else None
    L.check(lib.pgt_conv_rgb_bf16(_p(x_nchw), F, H, W, ksize, stride, pad, m, s, _p(wp), wp.stride(0), wp.shape[0],
                                  _p(bias), act, _p(out), _rows(out)[2], _p(gn_stats), _stream()))
    return out


def conv_up2x(x, wp4, cout, out, bias=None, act=ACT_NONE, gn_stats=None):
    """nearest x2 upsample + conv3x3 folded into four 2x2 phase convs; wp4 [4, cout, 4*CinPad] bf16."""
    lib = L.load()
    F, H, W, Cin = x.shape
    assert x.dtype == torch.bfloat16 and wp4.dtype == torch.bfloat16 and wp4.is_contiguous() and wp4.dim() == 3
    assert tuple(out.shape) == (F, 2 * H, 2 * W, cout) and out.is_contiguous()
    ep = make_epilogue(out, bias, act, gn_stats=gn_stats)
    L.check(lib.pgt_conv_up2x_bf16(_p(x), F, H, W, Cin, x.stride(2), _p(wp4), wp4.stride(1), cout, ctypes.byref(ep),
                                   _stream()))
    return out


_gn_ws = {}


def _gn_workspace(kind, x, n):
    """fp32 GroupNorm scratch of at least n floats, one per (kind, device, current stream), grown on demand: 'stats'
    holds pgt_groupnorm_ws_floats partial statistics, 'ab' the [F, 2, C] affine terms of groupnorm_apply_stats.

    Under CUDA-graph capture the scratch is a fresh tensor from the capturing graph's own memory pool and is not cached:
    a cached one would be shared by every graph captured on that stream and could be freed (grown, or released with
    the pool of a destroyed graph) while another graph still replays into it."""
    if torch.cuda.is_current_stream_capturing():
        return torch.empty(max(n, 1), dtype=torch.float32, device=x.device)
    key = (kind, x.device.index, torch.cuda.current_stream().cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < n:
        ws = torch.empty(max(n, 1 << 16), dtype=torch.float32, device=x.device)
        _gn_ws[key] = ws
    return ws


def groupnorm_silu(x, gamma, beta, out, eps=1e-6, silu=True):
    lib = L.load()
    F = x.shape[0]
    C = x.shape[-1]
    HW = x.numel() // (F * C) if x.is_contiguous() else x.shape[1] * x.shape[2]
    _, _, ldx = _rows(x)
    _, _, ldy = _rows(out)
    ws = _gn_workspace('stats', x, lib.pgt_groupnorm_ws_floats(F, HW, C))
    L.check(lib.pgt_groupnorm_silu(_p(x), ldx, F, HW, C, _p(gamma), _p(beta), eps, int(silu), _p(out), ldy, _p(ws),
                                   _stream()))
    return out


def conv_tiles_per_frame(H, W, cout, ksize=3, stride=1, pad_lo=1):
    return int(L.load().pgt_conv_tiles_per_frame(H, W, cout, ksize, stride, pad_lo))


def conv_tiles_exact(H, W, cout, ksize=3, stride=1, pad_lo=1):
    """conv_tiles_per_frame, or 0 when the tile grid does not divide the frame (the fused statistics would then include
    rows past the frame's edge)."""
    return int(L.load().pgt_conv_tiles_exact(H, W, cout, ksize, stride, pad_lo))


def groupnorm_apply_stats(x, gamma, beta, out, stats, chunks_per_frame, eps=1e-6, silu=True):
    """GroupNorm(32)+SiLU whose statistics were produced by the previous conv / linear epilogue."""
    lib = L.load()
    F = x.shape[0]
    C = x.shape[-1]
    HW = x.shape[1] * x.shape[2]
    ws = _gn_workspace('ab', x, F * 2 * C)
    L.check(lib.pgt_groupnorm_apply_stats(_p(x), _rows(x)[2], F, HW, C, _p(gamma), _p(beta), eps, int(silu), _p(out),
                                          _rows(out)[2], _p(stats), chunks_per_frame, _p(ws), _stream()))
    return out


def groupnorm_ab(x, gamma, beta, ab, stats=None, chunks_per_frame=0, eps=1e-6):
    """Per-(frame, channel) GroupNorm affine terms ab [F, 2, C] fp32 (for conv_out_gn), from fused statistics or from
    x."""
    lib = L.load()
    F = x.shape[0]
    C = x.shape[-1]
    HW = x.shape[1] * x.shape[2]
    ws = None if stats is not None else _gn_workspace('stats', x, lib.pgt_groupnorm_ws_floats(F, HW, C))
    assert ab.dtype == torch.float32 and ab.numel() >= F * 2 * C and ab.is_contiguous()
    L.check(lib.pgt_groupnorm_ab(_p(x), _rows(x)[2], F, HW, C, _p(gamma), _p(beta), eps, _p(stats), chunks_per_frame,
                                 _p(ws), _p(ab), _stream()))
    return ab


def conv_out_gn(x, ab, wp, cout, bias, out, silu=True):
    """conv3x3(silu(groupnorm(x))) -> fp32 NCHW for the decoder tail (Cin = 64 or 128, Cout <= 3); with silu=False
    conv3x3(groupnorm(x)) (VQGAN's generator tail).  None when not covered."""
    lib = L.load()
    F, H, W, Cin = x.shape
    assert x.dtype == torch.bfloat16 and x.stride(3) == 1 and x.stride(1) == W * x.stride(2) and \
        (F == 1 or x.stride(0) == H * x.stride(1))
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (F, cout, H, W)
    if silu:
        rc = lib.pgt_conv_out_gn(_p(x), F, H, W, Cin, x.stride(2), _p(ab), _p(wp), wp.stride(0), cout, _p(bias), _p(out),
                                 _stream(x))
    else:
        rc = lib.pgt_conv_out_gn_act(_p(x), F, H, W, Cin, x.stride(2), _p(ab), _p(wp), wp.stride(0), cout, _p(bias),
                                     _p(out), 0, _stream(x))
    if rc == -3:
        return None
    L.check(rc)
    return out


def layernorm(x, gamma, beta, out, eps=1e-5, pos=None, out2=None):
    lib = L.load()
    T, C, ldx = _rows(x)
    L.check(lib.pgt_layernorm(_p(x), ldx, _dt(x), T, C, _p(gamma), _p(beta), eps, _p(out), _rows(out)[2],
                              _p(pos), _rows(pos)[2] if pos is not None else 0,
                              _p(out2), _rows(out2)[2] if out2 is not None else 0, _stream()))
    return out


def ln_linear(x, ln_g, ln_b, w, bias, out, eps=1e-5):
    """out = LN(x) @ w^T + bias fused (C == 256, N % 256 == 0); x [..., 256] bf16, w [N, 256] bf16."""
    lib = L.load()
    T, C, ldx = _rows(x)
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.stride(1) == 1 and out.dtype == torch.bfloat16
    L.check(lib.pgt_ln_linear_bf16(_p(x), ldx, T, C, _p(ln_g), _p(ln_b), eps, _p(w), w.stride(0), w.shape[0], _p(bias),
                                   _p(out), _rows(out)[2], _stream()))
    return out


def swin_mlp(x, ln_g, ln_b, w1, b1, w2, b2, out, eps=1e-5, gn_stats=None):
    """out = x + fc2(gelu(fc1(LN(x)))) fused (C == 256); x, out: [..., C] bf16 with a uniform row stride."""
    lib = L.load()
    T, C, ldx = _rows(x)
    assert x.dtype == torch.bfloat16 and w1.dtype == torch.bfloat16 and w1.is_contiguous() and w2.is_contiguous()
    L.check(lib.pgt_swin_mlp_bf16(_p(x), ldx, T, C, _p(ln_g), _p(ln_b), eps, _p(w1), _p(b1), _p(w2), _p(b2), _p(out),
                                  _rows(out)[2], _p(gn_stats), _stream()))
    return out


def window_attention(qkv, clips, H, W, C, heads, shift, bias_tab, out):
    lib = L.load()
    assert qkv.dtype == torch.bfloat16 and bias_tab.dtype == torch.float32 and bias_tab.is_contiguous()
    L.check(lib.pgt_window_attention(_p(qkv), _rows(qkv)[2], clips, H, W, C, heads, shift, _p(bias_tab), _p(out),
                                     _rows(out)[2], _stream()))
    return out


LOG2E = 1.4426950408889634


def window_tables(bias):
    """Bias tables of pgt_window_attention_tc from the expanded relative-position bias [heads, 48, 48] fp32:
    fp16 [4 types][heads][6][48][8] = bias[pi(row)][pi(key)] * log2(e), where type 0 is an interior window, 1 / 2 / 3 a
    window that wraps in x / y / both (last window column / row of a shifted block): the TMA boxes of its halves land
    one after the other, which permutes the rows (pi).  The reference's {0, -100} shift mask
    (`modules/rstt_layers.py:552-568`), which separates tokens on different sides of the wrap, is not in the table: the
    kernel adds it in fp32 (in fp16, near -144, it would be rounded by up to 0.0625 in the log2 domain)."""
    heads = bias.shape[0]
    dev = bias.device
    r = torch.arange(48, device=dev)
    tabs = []
    for t in range(4):
        if t == 0:
            f, iy, ix = r // 16, (r // 4) % 4, r % 4
        elif t == 1:                                   # parts x in {W-2, W-1} then {0, 1}: rows [f][y][x(2)]
            rr = r % 24
            f, iy, ix = rr // 8, (rr % 8) // 2, rr % 2 + 2 * (r // 24)
        elif t == 2:                                   # parts y in {H-2, H-1} then {0, 1}: rows [f][y(2)][x]
            rr = r % 24
            f, iy, ix = rr // 8, (rr % 8) // 4 + 2 * (r // 24), rr % 4
        else:                                          # four quarter boxes, y outer / x inner: rows [f][y(2)][x(2)]
            pp, rr = r // 12, r % 12
            f, iy, ix = rr // 4, (rr % 4) // 2 + 2 * (pp // 2), rr % 2 + 2 * (pp % 2)
        canon = f * 16 + iy * 4 + ix
        tt = bias[:, canon][:, :, canon].float() * LOG2E                     # [heads, row, key]
        tabs.append(tt.view(heads, 48, 6, 8).permute(0, 2, 1, 3))             # [heads, 6, row, 8]
    return torch.stack(tabs, 0).to(torch.float16).contiguous()


def window_attention_tc(qkv, clips, H, W, C, heads, shift, tab16, out):
    """TMA + wgmma window attention core; returns None when the shape is not covered (caller uses window_attention)."""
    lib = L.load()
    assert qkv.dtype == torch.bfloat16 and tab16.dtype == torch.float16 and tab16.is_contiguous()
    rc = lib.pgt_window_attention_tc(_p(qkv), _rows(qkv)[2], clips, H, W, C, heads, shift, _p(tab16), _p(out),
                                     _rows(out)[2], _stream(qkv))
    if rc == -3:
        return None
    L.check(rc)
    return out


def window3d_attention(qkv, B, D, H, W, C, heads, window, shift, bias, out, pad_qkv=None):
    """Generic 3-D shifted-window attention core (Video-Swin BasicLayer of TDRQVAE); bias fp32 [heads, N, N]."""
    lib = L.load()
    assert qkv.dtype == torch.bfloat16 and bias.dtype == torch.float32 and bias.is_contiguous()
    L.check(lib.pgt_window3d_attention(_p(qkv), _rows(qkv)[2], _p(pad_qkv), B, D, H, W, C, heads, window[0], window[1],
                                       window[2], shift[0], shift[1], shift[2], _p(bias), _p(out), _rows(out)[2],
                                       _stream(qkv)))
    return out


def mha(q, k, v, clips, L_, heads, d, out):
    lib = L.load()
    L.check(lib.pgt_mha_fwd(_p(q), _rows(q)[2], _p(k), _rows(k)[2], _p(v), _rows(v)[2], clips, L_, heads, d, _p(out),
                            _rows(out)[2], _stream()))
    return out


def argmax_gather(logits, codebook, idx_out, quant, idx_in=None):
    """Row argmax of logits + codebook gather; with idx_in (int64, every entry a valid codebook row: the kernel does no
    range check) logits may be None and only the gather runs."""
    lib = L.load()
    if logits is None:
        assert idx_in is not None and idx_in.dtype == torch.int64 and idx_in.is_contiguous()
        T, K = idx_in.numel(), 4                       # K is not read when the codes are given
    else:
        T, K = logits.shape
        assert logits.dtype == torch.float32 and logits.is_contiguous()
    assert codebook.dtype == torch.float32
    assert idx_out is None or idx_out.dtype == torch.int64
    L.check(lib.pgt_argmax_gather(_p(logits), T, K, _p(codebook), codebook.shape[1], _p(idx_in), _p(idx_out),
                                  _p(quant), _rows(quant)[2] if quant is not None else 0,
                                  _dt(quant) if quant is not None else 0, _stream()))
    return idx_out, quant


def l2_argmin(z, codebook, K, idx_out, quant=None):
    lib = L.load()
    T, E = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous() and codebook.is_contiguous()
    L.check(lib.pgt_l2_argmin(_p(z), T, E, _p(codebook), K, _p(idx_out), _p(quant), _stream()))
    return idx_out, quant


def codebook_pack(codebook, K):
    """Load-time pack for l2_argmin_tc: (bf16 copy [K, E], fp32 [K + 2] = ||e_k||^2, max||e~||^2, max||e - e~||^2)."""
    lib = L.load()
    E = codebook.shape[1]
    assert codebook.dtype == torch.float32 and codebook.is_contiguous() and codebook.shape[0] >= K
    cb16 = torch.empty(K, E, dtype=torch.bfloat16, device=codebook.device)
    norm = torch.empty(K + 2, dtype=torch.float32, device=codebook.device)
    L.check(lib.pgt_codebook_pack(_p(codebook), K, E, _p(cb16), _p(norm), _stream(codebook)))
    return cb16, norm


L2_ARGMIN_UNSUPPORTED = -3
_last_argmin_ws = None


def last_l2_argmin_fallbacks():
    """Tokens of the last l2_argmin_tc call that went through the exhaustive kernel (diagnostics; synchronises)."""
    return int(_last_argmin_ws[0].item()) if _last_argmin_ws is not None else 0


def l2_argmin_tc(z, codebook, pack, K, idx_out, quant=None):
    """wgmma nearest-codebook argmin (exact, see l2_argmin_tc.cu); falls back to the exhaustive kernel for shapes the
    tensor-core kernel does not cover (K % 256, E % 128, E > 512)."""
    lib = L.load()
    T, E = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous() and codebook.is_contiguous() and idx_out.dtype == torch.int64
    global _last_argmin_ws
    ws = torch.empty(int(lib.pgt_l2_argmin_ws_ints(T)), dtype=torch.int32, device=z.device)
    _last_argmin_ws = ws
    rc = lib.pgt_l2_argmin_tc(_p(z), T, E, _p(codebook), _p(pack[0]), _p(pack[1]), K, _p(idx_out), _p(quant), _p(ws),
                              _stream(z))
    if rc == L2_ARGMIN_UNSUPPORTED:
        return l2_argmin(z, codebook, K, idx_out, quant)
    L.check(rc)
    return idx_out, quant


ARGMIN_MIN_CODES_PER_SPLIT = 512     # floor on codes per range of l2_argmin_tc_split (DESIGN §6, item 8)


def argmin_splits(T, K, device=None):
    """Code ranges for l2_argmin_tc_split: enough (token tile, range) CTAs to cover the SMs, min(K / 128, SMs / tiles),
    but no range below ARGMIN_MIN_CODES_PER_SPLIT codes; 1 once the token tiles alone fill the GPU."""
    sms = torch.cuda.get_device_properties(device if device is not None else torch.cuda.current_device()).multi_processor_count
    tiles = (T + 127) // 128
    return max(1, min(K // 128, sms // tiles, K // ARGMIN_MIN_CODES_PER_SPLIT))


def l2_argmin_tc_split(z, codebook, pack, K, idx_out, quant=None, splits=None):
    """l2_argmin_tc with the codebook split over `splits` code ranges (default argmin_splits(T, K)): the same codes, more
    CTAs at small T (l2_argmin_tc.cu).  K a multiple of 128, E a multiple of 128 up to 512."""
    lib = L.load()
    T, E = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous() and codebook.is_contiguous() and idx_out.dtype == torch.int64
    if splits is None:
        splits = argmin_splits(T, K, z.device)
    ws = torch.empty(int(lib.pgt_l2_argmin_split_ws_ints(T, int(splits))), dtype=torch.int32, device=z.device)
    L.check(lib.pgt_l2_argmin_tc_split(_p(z), T, E, _p(codebook), _p(pack[0]), _p(pack[1]), K, int(splits), _p(idx_out),
                                       _p(quant), _p(ws), _stream(z)))
    return idx_out, quant


def soft_codes(z, codebook, norm, K, temp, out):
    """out[T, K] = softmax_k(-||z - e_k||^2 / temp) over the first K codebook rows (soft_codes.cu); norm: the fp32
    ||e_k||^2 of codebook_pack.  out may be row-pitched (one depth's K-slice of a contiguous [T, D, K] tensor)."""
    lib = L.load()
    T, E = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous() and codebook.dtype == torch.float32 and codebook.is_contiguous()
    assert codebook.shape[1] == E and codebook.shape[0] >= K and norm.dtype == torch.float32 and norm.numel() >= K
    assert out.dtype == torch.float32 and tuple(out.shape) == (T, K) and out.stride(1) == 1
    L.check(lib.pgt_soft_codes(_p(z), T, E, _p(codebook), _p(norm), K, float(temp), _p(out), out.stride(0), _stream(z)))
    return out


def sample_codes(p, seed, idx_out):
    """idx_out[t] = one draw from the distribution in row t of p (codebook.cu sample_codes_kernel), p [T, K] possibly
    row-pitched; seed: device int64 [2] (Philox key and offset), read on the device; idx_out int64 [T] contiguous."""
    lib = L.load()
    T, K = p.shape
    assert p.dtype == torch.float32 and p.stride(1) == 1 and idx_out.dtype == torch.int64 and idx_out.numel() == T
    assert idx_out.is_contiguous() and seed.dtype == torch.int64 and seed.numel() == 2 and seed.device == p.device
    assert idx_out.device == p.device
    L.check(lib.pgt_sample_codes(_p(p), T, K, p.stride(0), _p(seed), _p(idx_out), _stream(p)))
    return idx_out


def rq_residual(r_in, r_out, idx, codebook, agg, first):
    """One residual-quantiser step (rq.cu): e = codebook[idx[t]]; r_out = r_in - e and agg = e if first else agg + e,
    each skipped when its output is None.  fp32 [T, E] contiguous; idx int64 [T] contiguous."""
    lib = L.load()
    ref = agg if agg is not None else r_out
    T, E = ref.shape
    assert codebook.dtype == torch.float32 and codebook.is_contiguous() and codebook.shape[1] == E
    assert idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == T and idx.device == ref.device
    for r in (r_in, r_out, agg):
        assert r is None or (r.dtype == torch.float32 and r.is_contiguous() and tuple(r.shape) == (T, E))
    L.check(lib.pgt_rq_residual(_p(r_in), _p(r_out), _p(idx), T, E, _p(codebook), _p(agg), int(bool(first)),
                                _stream(ref)))
    return agg


def rq_embed(idx, d0, d1, codebooks, out, ldi, ldd):
    """out[t] = sum_{d = d0..d1} codebooks[d or 0][idx[t * ldi + d * ldd]] (rq.cu); codebooks fp32 [D, K + 1, E], or
    [1, K + 1, E] for a codebook shared by every depth (read with depth stride 0).  out fp32 / bf16 [T, E] rows."""
    lib = L.load()
    T, E, ldo = _rows(out)
    assert codebooks.dtype == torch.float32 and codebooks.is_contiguous() and codebooks.dim() == 3 and codebooks.shape[2] == E
    assert idx.dtype == torch.int64 and idx.device == out.device and 0 <= d0 <= d1
    assert codebooks.shape[0] == 1 or d1 < codebooks.shape[0]
    assert idx.is_contiguous() and (T - 1) * ldi + d1 * ldd < idx.numel()
    cb_stride = 0 if codebooks.shape[0] == 1 else codebooks.shape[1] * E
    L.check(lib.pgt_rq_embed(_p(idx), ldi, ldd, T, d0, d1, _p(codebooks), cb_stride, E, _p(out), ldo, _dt(out),
                             _stream(out)))
    return out


def vq_stats(z, codebook, idx, HW, beta, scalars, zq_nchw=None, zq_bf16=None, min_enc=None, scores=None, usage=None):
    """VectorQuantizer.forward's outputs after the argmin (vq.cu): z fp32 [T, E] rows (T = b * HW), codebook fp32 [K, E],
    idx int64 [T].  Writes the straight-through z + (e - z) (fp32 NCHW [b, E, h, w] and / or bf16 [T, E] rows), the
    one-hot min_enc [T, K], scores [T], adds the counts to usage (int32 [K]) and writes scalars fp32 [3] = (loss,
    perplexity, mean_distance).  Outputs left None are not written."""
    lib = L.load()
    T, E = z.shape
    K = codebook.shape[0]
    assert z.dtype == torch.float32 and z.is_contiguous() and codebook.dtype == torch.float32 and codebook.is_contiguous()
    assert codebook.shape[1] == E and idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == T
    assert scalars.dtype == torch.float32 and scalars.numel() >= 3 and scalars.is_contiguous()
    assert zq_nchw is None or (zq_nchw.dtype == torch.float32 and zq_nchw.is_contiguous() and zq_nchw.numel() == T * E
                               and zq_nchw.shape[1] == E)
    assert zq_bf16 is None or (zq_bf16.dtype == torch.bfloat16 and zq_bf16.is_contiguous() and zq_bf16.numel() == T * E)
    assert min_enc is None or (min_enc.dtype == torch.float32 and min_enc.is_contiguous() and min_enc.numel() == T * K)
    assert scores is None or (scores.dtype == torch.float32 and scores.is_contiguous() and scores.numel() == T)
    assert usage is None or (usage.dtype == torch.int32 and usage.is_contiguous() and usage.numel() == K)
    for t in (idx, zq_nchw, zq_bf16, min_enc, scores, usage, scalars):
        assert t is None or t.device == z.device
    hist = torch.zeros(K, dtype=torch.int32, device=z.device)
    ws = torch.empty(max(int(lib.pgt_vq_stats_ws_doubles(T, E)), 1), dtype=torch.float64, device=z.device)
    L.check(lib.pgt_vq_stats(_p(z), T, E, int(HW), _p(codebook), K, _p(idx), float(beta), _p(zq_nchw), _p(zq_bf16),
                             _p(min_enc), _p(scores), _p(usage), _p(hist), _p(ws), _p(scalars), _stream(z)))
    return scalars


def adain(q, style, out, eps=1e-5, flags=None):
    """AdaIN of q [F, HW(, ...), C] against style into bf16 out; flags (device int32 [F]): frames whose flag is 0 are
    q rounded to bf16 instead (pgt_adain_frames)."""
    lib = L.load()
    F = q.shape[0]
    C = q.shape[-1]
    HW = q.shape[1] * q.shape[2] if q.dim() == 4 else q.shape[1]
    if flags is None:
        L.check(lib.pgt_adain(_p(q), _rows(q)[2], _dt(q), _p(style), _rows(style)[2], F, HW, C, eps, _p(out),
                              _rows(out)[2], _stream()))
        return out
    assert flags.dtype == torch.int32 and flags.is_contiguous() and flags.numel() == F and flags.device == q.device
    L.check(lib.pgt_adain_frames(_p(q), _rows(q)[2], _dt(q), _p(style), _rows(style)[2], F, HW, C, eps, _p(flags),
                                 _p(out), _rows(out)[2], _stream()))
    return out


def maxpool3x3s2(x, out):
    lib = L.load()
    F, H, W, C = x.shape
    L.check(lib.pgt_maxpool3x3s2(_p(x), _rows(x)[2], F, H, W, C, _p(out), _rows(out)[2], _stream()))
    return out


def global_avgpool(x, out):
    lib = L.load()
    F, H, W, C = x.shape
    L.check(lib.pgt_global_avgpool(_p(x), _rows(x)[2], F, H * W, C, _p(out), out.stride(0), _stream()))
    return out


def channel_affine(x, scale, out, plus_one=False, addv=None, addm=None):
    lib = L.load()
    F, H, W, C = x.shape
    L.check(lib.pgt_channel_affine(_p(x), _rows(x)[2], F, H * W, C, _p(scale), scale.stride(0), int(plus_one),
                                   _p(addv), addv.stride(0) if addv is not None else 0,
                                   _p(addm), _rows(addm)[2] if addm is not None else 0, _p(out), _rows(out)[2], _stream()))
    return out


def assemble_cond(o0, o1, o2, cond, ncls=19):
    lib = L.load()
    F, h8, w8, _ = o0.shape
    _, h16, w16, _ = o2.shape
    L.check(lib.pgt_assemble_cond(_p(o0), _rows(o0)[2], _p(o1), _rows(o1)[2], _p(o2), _rows(o2)[2], F, h8, w8, h16, w16,
                                  ncls, _p(cond), _rows(cond)[2], _stream()))
    return cond


def u8hwc_to_f32nchw(x_u8, out):
    """rgb24 frames [F,H,W,3] uint8 -> fp32 [F,3,H,W] = (float)(v / 255.0), numpy's rounding (inference.py:6-10)."""
    lib = L.load()
    F, H, W, C = x_u8.shape
    assert C == 3 and x_u8.dtype == torch.uint8 and x_u8.is_contiguous() and x_u8.is_cuda
    assert out.dtype == torch.float32 and tuple(out.shape) == (F, 3, H, W) and out.is_contiguous()
    L.check(lib.pgt_u8hwc_to_f32nchw(_p(x_u8), F, H, W, _p(out), _stream()))
    return out


def u8hwc_resize_to_f32nchw(x_u8, out, hw, sizes=None):
    """rgb24 source frames -> fp32 out [F,3,H,W]: (float)(v / 255.0), then bilinear with align_corners=True to H x W,
    bit for bit what F.interpolate gives on an AVX2 / AVX512 host (data/vfhq_full_dataset.py:1046-1051).  x_u8: uint8
    on the device holding the frames.  sizes None: every frame is hw = (h, w), packed one after another from x_u8's
    first byte.  sizes: device int32 [F, 3] of each frame's (h, w, byte offset from x_u8's first byte); hw then bounds
    them and only sizes the profile's byte count."""
    lib = L.load()
    F, C, H, W = out.shape
    h, w = hw
    assert x_u8.dtype == torch.uint8 and x_u8.is_contiguous() and x_u8.is_cuda
    assert C == 3 and out.dtype == torch.float32 and out.is_contiguous() and out.device == x_u8.device
    if sizes is None:
        assert x_u8.numel() >= F * h * w * 3
    else:
        assert sizes.dtype == torch.int32 and sizes.is_contiguous() and sizes.numel() == 3 * F and \
            sizes.device == x_u8.device
    L.check(lib.pgt_u8hwc_resize_to_f32nchw(_p(x_u8), F, h, w, _p(sizes), H, W, _p(out), _stream()))
    return out


def f32nchw_resize_to_f32nchw(x, out):
    """fp32 frames x [F,3,h,w] -> fp32 out [F,3,H,W] (H, W multiples of 64): bilinear with align_corners=True in the
    fma form of u8hwc_resize_to_f32nchw, the second step of the test set's `lr` degradation
    (data/vfhq_full_dataset.py:1017-1024)."""
    lib = L.load()
    F, C, h, w = x.shape
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous() and x.is_cuda
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape[:2]) == (F, 3) and \
        out.device == x.device
    L.check(lib.pgt_f32nchw_resize_to_f32nchw(_p(x), F, h, w, out.shape[2], out.shape[3], _p(out), _stream()))
    return out


def imresize_u8hwc_to_f32nchw(x_u8, taps_h, taps_w, out):
    """rgb24 frames x_u8 [F,h,w,3] on the device -> fp32 out [F,3,oh,ow]: basicsr's antialiased bicubic imresize of
    (float)(v / 255.0), each pass rounded once from its exact sum (pgt_imresize_u8hwc_to_f32nchw).  taps_h, taps_w:
    (weights fp32, indices int32), each [out, K] on the device, as pgtformer_b200.degrade builds them."""
    lib = L.load()
    F, h, w, C = x_u8.shape
    (wh, ih), (ww, iw) = taps_h, taps_w
    assert C == 3 and x_u8.dtype == torch.uint8 and x_u8.is_contiguous() and x_u8.is_cuda
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (F, 3, wh.shape[0], ww.shape[0])
    for t, dt in ((wh, torch.float32), (ih, torch.int32), (ww, torch.float32), (iw, torch.int32)):
        assert t.dtype == dt and t.dim() == 2 and t.is_contiguous() and t.device == x_u8.device
    L.check(lib.pgt_imresize_u8hwc_to_f32nchw(_p(x_u8), F, h, w, _p(wh), _p(ih), wh.shape[1], wh.shape[0], _p(ww),
                                              _p(iw), ww.shape[1], ww.shape[0], _p(out), _stream()))
    return out


def f32nchw_to_u8hwc(x, out_u8, first=0, step=1):
    """uint8(clamp(x, 0, 1) * 255) of frames first, first+step, ... -> rgb24 [n,H,W,3] (inference.py:15-19)."""
    lib = L.load()
    n, H, W, C = out_u8.shape
    assert C == 3 and out_u8.dtype == torch.uint8 and out_u8.is_contiguous()
    assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[1:] == (3, H, W) and first + (n - 1) * step < x.shape[0]
    L.check(lib.pgt_f32nchw_to_u8hwc(_p(x), first, step, n, H, W, _p(out_u8), _stream()))
    return out_u8


def gather_frames(x, idx_i32, out):
    """out[f] = x[idx[f]] along dim 0 (whole frames; idx: device int32)."""
    lib = L.load()
    assert x.is_contiguous() and out.is_contiguous() and x.dtype == out.dtype and x.shape[1:] == out.shape[1:]
    assert idx_i32.dtype == torch.int32 and idx_i32.is_cuda and idx_i32.numel() == out.shape[0]
    fb = x[0].numel() * x.element_size()
    L.check(lib.pgt_gather_frames(_p(x), fb, _p(idx_i32), out.shape[0], _p(out), _stream()))
    return out


def scatter_frames(x, idx_i32, out):
    """out[idx[f]] = x[f] along dim 0 (whole frames; idx: device int32, distinct entries) — gather_frames' mirror."""
    lib = L.load()
    assert x.is_contiguous() and out.is_contiguous() and x.dtype == out.dtype and x.shape[1:] == out.shape[1:]
    assert idx_i32.dtype == torch.int32 and idx_i32.is_cuda and idx_i32.numel() == x.shape[0]
    fb = x[0].numel() * x.element_size()
    L.check(lib.pgt_scatter_frames(_p(x), fb, _p(idx_i32), x.shape[0], _p(out), _stream()))
    return out


def frame_scores(a_u8, b_u8, sse=None, ssim=None):
    """PSNR / SSIM sums of F rgb24 frame pairs a_u8, b_u8 [F,H,W,3] uint8 on the device, H, W >= 11 (pgt_frame_scores):
    sse int64 [F], the exact sum of (a - b)^2 over all H W 3 values, and ssim fp64 [F,3], each channel's SSIM map mean
    (basicsr's calculate_ssim with crop_border 0; oracle/metrics_oracle.py).  Deterministic, and capture-safe: the
    workspace comes from the current allocator (a graph's own pool under capture)."""
    lib = L.load()
    F, H, W, C = a_u8.shape
    assert C == 3 and a_u8.dtype == torch.uint8 and a_u8.is_contiguous() and a_u8.is_cuda
    assert b_u8.shape == a_u8.shape and b_u8.dtype == torch.uint8 and b_u8.is_contiguous() and b_u8.device == a_u8.device
    if sse is None:
        sse = torch.empty(F, dtype=torch.int64, device=a_u8.device)
    if ssim is None:
        ssim = torch.empty(F, 3, dtype=torch.float64, device=a_u8.device)
    assert sse.dtype == torch.int64 and sse.is_contiguous() and sse.numel() == F and sse.device == a_u8.device
    assert ssim.dtype == torch.float64 and ssim.is_contiguous() and ssim.numel() == 3 * F and ssim.device == a_u8.device
    ws = torch.empty(max(int(lib.pgt_frame_scores_ws_doubles(F, H, W)), 1), dtype=torch.float64, device=a_u8.device)
    L.check(lib.pgt_frame_scores(_p(a_u8), _p(b_u8), F, H, W, _p(ws), _p(sse), _p(ssim), _stream(a_u8)))
    return sse, ssim


def copy2d(x, out):
    lib = L.load()
    T, C, ldx = _rows(x)
    L.check(lib.pgt_copy2d(_p(x), ldx, T, C, _p(out), _rows(out)[2], _stream()))
    return out


def regroup_frames(x, out, clips, P, C, direction):
    lib = L.load()
    L.check(lib.pgt_regroup_frames(_p(x), _rows(x)[2], clips, P, C, _p(out), _rows(out)[2], direction, _stream()))
    return out


def nchw_to_nhwc(x, out, mean=None, std=None):
    lib = L.load()
    F, C, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    L.check(lib.pgt_nchw_f32_to_nhwc_bf16(_p(x), F, C, H * W, _p(mean), _p(std), _p(out), _rows(out)[2], _stream()))
    return out


def nhwc_to_f32(x, out, to_nchw):
    lib = L.load()
    F, H, W, C = x.shape
    L.check(lib.pgt_nhwc_bf16_to_f32(_p(x), _rows(x)[2], F, H * W, C, _p(out), int(to_nchw), _stream()))
    return out


def launch_count():
    return int(L.load().pgt_launch_count())


def reset_launch_count():
    L.load().pgt_reset_launch_count()


PROF_CLASSES = ('gemm_tc', 'window_attn', 'mha', 'argmax_gather', 'l2_argmin', 'groupnorm', 'move', 'layernorm')


def profile_begin():
    L.check(L.load().pgt_profile_begin())


def profile_end(csv_path=None):
    """-> {class: (work, ms, launches)}; work is FLOPs (gemm/attention/argmin) or bytes (argmax/norm).
    With csv_path, one row per launch is written there as well."""
    n = len(PROF_CLASSES)
    work, ms, cnt = (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_int64 * n)()
    if csv_path is None:
        L.check(L.load().pgt_profile_end(work, ms, cnt))
    else:
        L.check(L.load().pgt_profile_end_csv(csv_path.encode(), work, ms, cnt))
    return {PROF_CLASSES[i]: (work[i], ms[i], int(cnt[i])) for i in range(n)}
