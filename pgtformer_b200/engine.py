"""H100 forward engine for PGTFormer: one-time weight repack into kernel layouts + the launch
sequence of `PGTFormer.forward` / `TDCRQVAE3.forward` over libpgt_b200.so.

Data layout in HBM (DESIGN.md §3): every activation is channels-last bf16 — feature maps
[F=clips*3, H, W, C], token matrices [T, C] — except the tensors the reference returns
(`out` fp32 NCHW, `logits` fp32, `lq_feat` fp32 NHWC) and the residual stream of the 9-layer global
transformer (fp32, it decides the code indices).  Frames of a clip are contiguous, so the
frame-major token order of the global transformer (`archs/pgtformer_arch.py:614,640`) is the
natural row order and no permute is ever materialised.

Every op — including the BiSeNet parsing net, whose eval-mode BatchNorms are folded at load time — is a call
into the C ABI; there is no PyTorch / cuDNN / CPU fallback: without the CUDA library construction fails.
"""
import os

import torch
import torch.nn.functional as F  # noqa: F401  (load-time weight padding only)

from . import ops
from .spec import Arch

BF = torch.bfloat16


def _on_device(fn):
    """Runs an Engine entry point with the engine's GPU as the current CUDA device: the C ABI launches on the current
    device's current stream, and its per-device one-time setup (kernel attributes, constant tables) keys on it, so a model
    on cuda:1 must not launch while cuda:0 is current."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        with torch.cuda.device(self.dev):
            return fn(self, *a, **k)
    return wrapper


def _pack_conv(w):
    """OIHW fp32 -> [Cout, k*k*CinPad] bf16 (K index = tap*CinPad + c)."""
    co, ci, kh, kw = w.shape
    cp = (ci + 63) // 64 * 64
    wp = torch.zeros(co, kh * kw, cp, dtype=torch.float32, device=w.device)
    wp[:, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return wp.reshape(co, kh * kw * cp).to(BF).contiguous()


def fold_layernorm_affine(weight, bias, gamma, beta):
    """(x_hat * gamma + beta) W^T + c  ==  x_hat (W * gamma)^T + (W beta + c), x_hat = (x - mean) * rstd: the affine of a
    LayerNorm folded into the linear layer that consumes it (norm1 -> q/kv and norm2 -> fc1 of the C = 256 Swin blocks,
    `modules/rstt_layers.py:298-336`), so that the fused kernels only normalise.  fp32 in, fp32 out (the caller rounds the
    folded weight to bf16 once).  Returns (W * gamma [N, C], W beta + c [N])."""
    wf = weight.float()
    return wf * gamma.float()[None, :], (bias.float() + wf @ beta.float()).contiguous()


def _pack_up2x(w):
    """OIHW 3x3 fp32 -> [4, Cout, 4*CinPad] bf16 phase weights of the upsample-folded conv (include/pgt_b200.h):
    phase (py,px), tap (ty,tx) = sum of w[dy,dx] over dy in S(py,ty), dx in S(px,tx); sums in fp32, one bf16 rounding."""
    co, ci, _, _ = w.shape
    cp = (ci + 63) // 64 * 64
    sets = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    out = torch.zeros(4, co, 4, cp, dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    acc = torch.zeros(co, ci, dtype=torch.float32, device=w.device)
                    for dy in sets[py][ty]:
                        for dx in sets[px][tx]:
                            acc += w[:, :, dy, dx]
                    out[py * 2 + px, :, ty * 2 + tx, :ci] = acc
    return out.reshape(4, co, 4 * cp).to(BF).contiguous()


def _pack_lin(w):
    """[N, K] (or [N, K, 1, 1]) fp32 -> [N, roundup(K, 8)] bf16."""
    w = w.reshape(w.shape[0], -1)
    n, k = w.shape
    kp = (k + 7) // 8 * 8
    if kp != k:
        w = F.pad(w, (0, kp - k))
    return w.to(BF).contiguous()


def _pack_rgb(w):
    """[Cout, 3, k, k] fp32 -> [Cout, roundup(3*k*k, 8)] bf16 with K index (ky*k + kx)*3 + c (ops.im2col_rgb order)."""
    return _pack_lin(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))


class Engine:
    arch_class = Arch

    def __init__(self, network_g, state_dict, device):
        ops.L.load()                                   # fail loudly if the CUDA library is missing
        self.arch = self.arch_class(network_g)
        self.dev = torch.device(device)
        if self.dev.type != 'cuda':
            raise RuntimeError('pgtformer_b200 has no CPU path: the engine needs a CUDA (sm_90a) device')
        self.w = {}
        with torch.cuda.device(self.dev):
            self._sd = {k: v.detach().to(self.dev) for k, v in state_dict.items()}
            self._repack()

    # ------------------------------------------------------------------ weight repack (load time)
    def _f32(self, name):
        return self._sd[name].float().contiguous()

    def _repack(self):
        sd, w = self._sd, self.w
        for name, t in sd.items():
            if name.startswith('conditionnet.'):
                continue
            if name.endswith('.weight') and t.dim() == 4:
                if name == 'encoder.conv_in.weight':
                    w[name] = _pack_rgb(t.float())
                elif t.shape[2] == 3 and '.upsample.conv.' in name:
                    w[name] = _pack_up2x(t.float())
                elif t.shape[2] == 3:
                    w[name] = _pack_conv(t.float())
                else:
                    w[name] = _pack_lin(t.float())
            elif name.endswith('.weight') and t.dim() == 2 and 'codebooks' not in name:
                w[name] = _pack_lin(t.float())
            elif t.dtype.is_floating_point and t.dim() == 1:
                w[name] = t.float().contiguous()
        w['codebook'] = self._f32('quantizer.codebooks.0.weight')
        if self.depth > 1:
            # every distinct codebook stacked once [D or 1, K + 1, E] (rq_embed reads a shared one with depth stride 0)
            n = 1 if self.arch.shared_codebook else self.depth
            w['codebooks'] = torch.stack([self._f32('quantizer.codebooks.%d.weight' % d) for d in range(n)]).contiguous()
        # Swin blocks: fused [q | k | v] projection and the expanded relative-position bias
        for name in list(sd):
            if name.endswith('.attn.relative_position_bias_table'):
                p = name[:-len('.relative_position_bias_table')]
                heads = sd[name].shape[1]
                idx = sd[p + '.relative_position_index'].view(-1).long()
                w[p + '.bias_tab'] = sd[name].float()[idx].view(48, 48, heads).permute(2, 0, 1).contiguous()
                w[p + '.tab16'] = ops.window_tables(w[p + '.bias_tab'])     # wgmma window kernel: bias, 4 box layouts
                w[p + '.qkv.weight'] = _pack_lin(torch.cat([sd[p + '.q.weight'], sd[p + '.kv.weight']], 0).float())
                w[p + '.qkv.bias'] = torch.cat([sd[p + '.q.bias'], sd[p + '.kv.bias']], 0).float().contiguous()
                blk = p[:-len('.attn')]
                if self.fuse_ln_qkv and sd[p + '.q.weight'].shape[1] == 256 and (blk + '.norm1.weight') in sd:
                    # norm1's affine folded into the projection the fused kernel applies to the normalised tile:
                    # (xh * g + b) W^T + c = xh (W * g)^T + (W b + c); products and sums in fp32, one bf16 rounding of W * g
                    wf = torch.cat([sd[p + '.q.weight'], sd[p + '.kv.weight']], 0)
                    wg, bg = fold_layernorm_affine(wf, w[p + '.qkv.bias'], sd[blk + '.norm1.weight'], sd[blk + '.norm1.bias'])
                    w[p + '.qkv_ln.weight'], w[p + '.qkv_ln.bias'] = _pack_lin(wg), bg
        # global transformer: in_proj split into the (q,k) projection of LN(x)+pos and the v projection of LN(x)
        E = self.arch.dim_embd
        for i in range(self.arch.n_layers):
            p = 'ft_layers.%d.self_attn' % i
            wi, bi = sd[p + '.in_proj_weight'].float(), sd[p + '.in_proj_bias'].float()
            w[p + '.qk.weight'], w[p + '.qk.bias'] = _pack_lin(wi[:2 * E]), bi[:2 * E].contiguous()
            w[p + '.v.weight'], w[p + '.v.bias'] = _pack_lin(wi[2 * E:]), bi[2 * E:].contiguous()
        # Swin MLP halves: norm2's affine folded into fc1 (same algebra as norm1 -> q/kv above)
        if self.fuse_swin_mlp:
            for name in list(sd):
                if name.endswith('.mlp.fc1.weight') and sd[name].shape == (256, 256):
                    blk = name[:-len('.mlp.fc1.weight')]
                    if (blk + '.norm2.weight') not in sd:
                        continue
                    wg, bg = fold_layernorm_affine(sd[name], sd[blk + '.mlp.fc1.bias'], sd[blk + '.norm2.weight'],
                                                   sd[blk + '.norm2.bias'])
                    w[blk + '.mlp.fc1_ln.weight'], w[blk + '.mlp.fc1_ln.bias'] = _pack_lin(wg), bg
        self._repack_parsing()

    # ------------------------------------------------------------------ small helpers
    @property
    def depth(self):
        """Quantiser depth D = code_shape[2]: codes per token."""
        return int(self.arch.code_shape[2])

    def _new(self, *shape, dtype=BF):
        return torch.empty(*shape, dtype=dtype, device=self.dev)

    fuse_cat_in_place = True  # SFT concat: encoder / decoder level outputs written straight into the concat buffer
    _fusing = False           # set per forward: SFT fusion active (w > 0)
    fuse_conv_out = True      # decoder norm_out + SiLU + conv_out (64 -> 3) as one kernel (conv_out.cu)
    window_tc = True          # window attention core on TMA + wgmma (window_attn_tc.cu)
    fuse_ln_qkv = True        # norm1 + q/kv projection of the C=256 Swin blocks as one kernel
    fuse_swin_mlp = True      # LN + fc1 + GELU + fc2 + residual of the C=256 Swin blocks as one kernel
    # GroupNorm+SiLU applied inside the consuming 3x3 conv (pgt_conv_gn_bf16, bit-identical).  Off by default: the
    # narrow (Cout <= 128) halo convs are bound by shared-memory operand reads, so the in-place slab transform costs
    # them more (+10 ms at 16 clips of 512^2) than the GroupNorm apply passes it removes (-6.8 ms); see DESIGN.md.
    fuse_gn_apply = os.environ.get('PGT_FUSE_GN', '') != ''
    fuse_gn_min_hw = int(os.environ.get('PGT_FUSE_GN', '0') or 0)       # fuse only for feature maps at least this tall
    fuse_gn_stats = True      # GroupNorm statistics from the producing conv / linear epilogue (saves one pass)

    def _stats_tiles(self, H, W, cout, ksize, stride, pad_lo):
        """Tiles per frame of a conv whose epilogue emits the next GroupNorm's statistics; 0: no fused statistics."""
        return ops.conv_tiles_per_frame(H, W, cout, ksize, stride, pad_lo)

    def _gn(self, x, p, silu=True):
        gn = getattr(x, '_pgt_gn', None)
        if gn is not None:
            return ops.groupnorm_apply_stats(x, self.w[p + '.weight'], self.w[p + '.bias'], self._new(*x.shape), gn[0], gn[1],
                                             silu=silu)
        return ops.groupnorm_silu(x, self.w[p + '.weight'], self.w[p + '.bias'], self._new(*x.shape), silu=silu)

    def _conv3(self, x, p, cout, out=None, gn_out=False, gn=None, gn_silu=True, **kw):
        """3x3 conv; gn: name of the Normalize() whose GroupNorm+SiLU precedes it — applied inside the conv kernel
        where the halo path exists (the normalised tensor never reaches HBM), as a separate pass otherwise.  With
        gn_silu=False the GroupNorm has no SiLU after it (VQGAN's encoder tail); the fused kernel always applies SiLU,
        so that case takes the separate pass."""
        Fr, H, W, cin = x.shape
        stride = kw.get('stride', 1)
        fused_ab = None
        if gn is not None:
            if gn_silu and self.fuse_gn_apply and H >= self.fuse_gn_min_hw and stride == 1 and kw.get('ksize', 3) == 3 and kw.get('pad_lo', 1) == 1 and \
                    'act' not in kw and not kw.get('relu_after_res') and ops.conv_gn_supported(H, W, cin, cout):
                st = getattr(x, '_pgt_gn', None)
                fused_ab = ops.groupnorm_ab(x, self.w[gn + '.weight'], self.w[gn + '.bias'],
                                            self._new(Fr * 2 * cin, dtype=torch.float32),
                                            stats=st[0] if st else None, chunks_per_frame=st[1] if st else 0)
            else:
                x = self._gn(x, gn, silu=gn_silu)
        if out is None:
            out = self._new(Fr, H // stride, W // stride, cout)
        stats = None
        if gn_out and self.fuse_gn_stats and cout % 32 == 0 and cout // 32 in (2, 4, 8, 16, 32) and out.is_contiguous():
            tpf = self._stats_tiles(H, W, cout, kw.get('ksize', 3), stride, kw.get('pad_lo', 1))
            if tpf > 0:
                stats = self._new(Fr * tpf * 4 * 64, dtype=torch.float32)      # [tile][32-row quadrant][32 groups][2]
                out._pgt_gn = (stats, tpf * 4)
        if fused_ab is not None:
            kw.pop('ksize', None); kw.pop('stride', None); kw.pop('pad_lo', None)
            return ops.conv_gn(x, fused_ab, self.w[p + '.weight'], cout, out, bias=self.w.get(p + '.bias'),
                               gn_stats=stats, **kw)
        return ops.conv(x, self.w[p + '.weight'], cout, out, bias=self.w.get(p + '.bias'), gn_stats=stats, **kw)

    def _lin(self, x, p, n, out=None, out_dtype=BF, gn_out=False, **kw):
        if out is None:
            out = self._new(*x.shape[:-1], n, dtype=out_dtype)
        stats = None
        if gn_out and self.fuse_gn_stats and out.dim() == 4 and out.dtype == BF and n % 32 == 0 and \
                n // 32 in (2, 4, 8, 16, 32) and (out.shape[1] * out.shape[2]) % 128 == 0 and out.is_contiguous():
            tpf = out.shape[1] * out.shape[2] // 128
            stats = self._new(out.shape[0] * tpf * 4 * 64, dtype=torch.float32)
            out._pgt_gn = (stats, tpf * 4)
        return ops.linear(x, self.w[p + '.weight'], out, bias=self.w.get(p + '.bias'), N=n, gn_stats=stats, **kw)

    # ------------------------------------------------------------------ blocks
    def td_resblock(self, x, p, cout, gn_next=False, out=None, shortcut='nin_shortcut'):
        """TDResnetBlock (`modules/rstt_layers.py:875-904`) / VQGAN's ResBlock (`archs/vqgan_arch.py:155-178`,
        shortcut='conv_out'): 2 x (GN+SiLU -> conv3x3), residual in the second conv's epilogue (the 1x1 shortcut first
        when the width changes).  conv1's epilogue also emits the GroupNorm statistics norm2 needs; with gn_next the
        block output carries them for the next Normalize()."""
        h = self._conv3(x, p + '.conv1', cout, gn=p + '.norm1', gn_out=True)
        sc = self._lin(x, p + '.' + shortcut, cout) if (p + '.' + shortcut + '.weight') in self.w else x
        return self._conv3(h, p + '.conv2', cout, gn=p + '.norm2', residual=sc, gn_out=gn_next, out=out)

    def swin_block(self, x, p, heads, shift, gn_next=False, out=None):
        """VSTSREncoderTransformerBlock (`modules/rstt_layers.py:284-338`) on [F,H,W,C]."""
        Fr, H, W, C = x.shape
        w = self.w
        if C == 256 and self.fuse_ln_qkv:
            # norm1 + the fused q/kv projection in one kernel (LN applied to the tile in shared memory)
            if (p + '.attn.qkv_ln.weight') in w:      # gamma / beta already inside the weights (see _repack)
                qkv = ops.ln_linear(x, None, None, w[p + '.attn.qkv_ln.weight'], w[p + '.attn.qkv_ln.bias'],
                                    self._new(Fr, H, W, 3 * C))
            else:
                qkv = ops.ln_linear(x, w[p + '.norm1.weight'], w[p + '.norm1.bias'], w[p + '.attn.qkv.weight'],
                                    w[p + '.attn.qkv.bias'], self._new(Fr, H, W, 3 * C))
        else:
            y = ops.layernorm(x, w[p + '.norm1.weight'], w[p + '.norm1.bias'], self._new(Fr, H, W, C))
            qkv = self._lin(y, p + '.attn.qkv', 3 * C)
        a = self._new(Fr, H, W, C)
        if not self.window_tc or ops.window_attention_tc(qkv, Fr // 3, H, W, C, heads, shift, w[p + '.attn.tab16'], a) is None:
            ops.window_attention(qkv, Fr // 3, H, W, C, heads, shift, w[p + '.attn.bias_tab'], a)   # shapes the TMA kernel does not cover
        x = self._lin(a, p + '.attn.proj', C, residual=x)
        if C == 256 and self.fuse_swin_mlp:
            # norm2 + fc1 + GELU + fc2 + residual in one kernel (the hidden tile never leaves the SM)
            out = self._new(Fr, H, W, C) if out is None else out
            stats = None
            if gn_next and self.fuse_gn_stats and (H * W) % 128 == 0 and out.is_contiguous():
                tpf = H * W // 128
                stats = self._new(Fr * tpf * 4 * 64, dtype=torch.float32)
                out._pgt_gn = (stats, tpf * 4)
            if (p + '.mlp.fc1_ln.weight') in w:       # gamma / beta already inside fc1 (see _repack)
                return ops.swin_mlp(x, None, None, w[p + '.mlp.fc1_ln.weight'], w[p + '.mlp.fc1_ln.bias'],
                                    w[p + '.mlp.fc2.weight'], w[p + '.mlp.fc2.bias'], out, gn_stats=stats)
            return ops.swin_mlp(x, w[p + '.norm2.weight'], w[p + '.norm2.bias'], w[p + '.mlp.fc1.weight'],
                                w[p + '.mlp.fc1.bias'], w[p + '.mlp.fc2.weight'], w[p + '.mlp.fc2.bias'], out,
                                gn_stats=stats)
        y = ops.layernorm(x, w[p + '.norm2.weight'], w[p + '.norm2.bias'], self._new(Fr, H, W, C))
        m = self._lin(y, p + '.mlp.fc1', C, act=ops.ACT_GELU)
        return self._lin(m, p + '.mlp.fc2', C, residual=x, gn_out=gn_next, out=out)

    def _repack_attn_qkv(self):
        """AttnBlock: q, k and v (1x1 convs of the same normalised input) as one [3C, C] projection."""
        sd, w = self._sd, self.w
        for name in list(sd):
            if name.endswith('.proj_out.weight'):
                p = name[:-len('.proj_out.weight')]
                w[p + '.qkv.weight'] = _pack_lin(torch.cat([sd[p + '.%s.weight' % n] for n in 'qkv'], 0).float())
                w[p + '.qkv.bias'] = torch.cat([sd[p + '.%s.bias' % n] for n in 'qkv'], 0).float().contiguous()

    def attn_block(self, x, p, gn_next=False):
        """AttnBlock (`archs/tdrqvae_arch.py:179-203`, `archs/vqgan_arch.py:181-240`): GroupNorm (no SiLU) -> q | k | v
        -> softmax(q k^T C^-1/2) v over all H*W tokens of each frame (one head of width C) -> proj_out + x.  The
        GroupNorm statistics come from the producing epilogue; with gn_next the output carries them for the next
        Normalize()."""
        Fr, H, W, C = x.shape
        y = self._gn(x, p + '.norm', silu=False)
        qkv = self._lin(y, p + '.qkv', 3 * C)
        a = ops.mha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], Fr, H * W, 1, C, self._new(Fr, H, W, C))
        return self._lin(a, p + '.proj_out', C, residual=x, gn_out=gn_next)

    def encoder_layer(self, x, p, heads, depth, gn_next=False, out=None):
        for i in range(depth):
            x = self.swin_block(x, '%s.blocks.%d' % (p, i), heads, 2 if i % 2 == 1 else 0,
                                gn_next=gn_next and i == depth - 1, out=out if i == depth - 1 else None)
        return x

    def _cat_slot(self, Fr, H, W, C):
        """Concat buffer [enc | dec | temporal] of a Fuse_sft_block level (`archs/pgtformer_arch.py:474`): the encoder
        level and, later, the decoder level write their outputs straight into its channel slices, so `torch.cat` costs
        no copy."""
        return self._new(Fr, H, W, 2 * C + 32)

    def fuse_sft(self, enc, dec, key, wgt, gn_next=False):
        """Fuse_sft_block (`archs/pgtformer_arch.py:460-484`); the final
        dec + w*(dec*scale + shift) is the epilogue of the last `shift` conv."""
        p = 'fuse_convs_dict.' + key
        Fr, H, W, C = dec.shape
        b, P = Fr // 3, H * W
        cat = getattr(enc, '_pgt_cat', None)
        if cat is None or getattr(dec, '_pgt_cat', None) is not cat:
            cat = self._new(Fr, H, W, 2 * C + 32)                # streaming gather / foreign tensors: copy into place
            ops.copy2d(enc, cat[..., :C])
            ops.copy2d(dec, cat[..., C:2 * C])
        tcat = self._new(b, P, 192)
        ops.regroup_frames(self._lin(enc, p + '.tconvenc', 32), tcat[..., :96], b, P, 32, 0)
        ops.regroup_frames(self._lin(dec, p + '.tconvdec', 32), tcat[..., 96:], b, P, 32, 0)
        fut = ops.regroup_frames(self._lin(tcat, p + '.tfusion0', 96), self._new(Fr, P, 32), b, P, 32, 1)
        self._lin(fut, p + '.tfusion1', 32, out=cat.view(Fr, P, 2 * C + 32)[..., 2 * C:])
        return self.sft_tail(cat, dec, p, wgt, gn_next)

    def sft_tail(self, cat, dec, p, wgt, gn_next=False):
        """The part of Fuse_sft_block PGTFormer (`archs/pgtformer_arch.py:476-484`) and CodeFormer
        (`archs/codeformer_arch.py:218-226`) share: encode_enc (ResBlock of the concat, 1x1 conv_out shortcut) ->
        scale / shift branches -> dec + w*(dec*scale + shift) in the epilogue of the last `shift` conv."""
        C = dec.shape[-1]
        e = p + '.encode_enc'
        h = self._conv3(cat, e + '.conv1', C, gn=e + '.norm1', gn_out=True)
        sc = self._lin(cat, e + '.conv_out', C)
        ef = self._conv3(h, e + '.conv2', C, gn=e + '.norm2', residual=sc)
        scale = self._conv3(self._conv3(ef, p + '.scale.0', C, act=ops.ACT_LRELU02), p + '.scale.2', C)
        sh = self._conv3(ef, p + '.shift.0', C, act=ops.ACT_LRELU02)
        return self._conv3(sh, p + '.shift.2', C, residual=dec, sft_scale=scale, sft_w=wgt, gn_out=gn_next)

    # ------------------------------------------------------------------ parsing net (BiSeNet / ResNet18)
    def _repack_parsing(self):
        """Eval-mode BatchNorm folded into the preceding conv (w' = w*g/sqrt(v+eps), b' = beta - mean*g/sqrt(v+eps)),
        then the usual kernel layouts (`archs/pgtformer_arch.py:40-397`)."""
        sd, w = self._sd, self.w
        P = 'conditionnet.'

        def fold(conv, bn):
            wt = sd[P + conv + '.weight'].float()
            if bn is None:
                return wt, None
            g, b = sd[P + bn + '.weight'].float(), sd[P + bn + '.bias'].float()
            m, v = sd[P + bn + '.running_mean'].float(), sd[P + bn + '.running_var'].float()
            s = g / torch.sqrt(v + 1e-5)
            return wt * s.view(-1, 1, 1, 1), (b - m * s).contiguous()

        def put(key, conv, bn, kind):
            wt, bias = fold(conv, bn)
            w['bn.' + key + '.weight'] = {'c3': _pack_conv, 'up': _pack_up2x, 'lin': _pack_lin,
                                          'rgb': _pack_rgb}[kind](wt)
            if bias is not None:
                w['bn.' + key + '.bias'] = bias

        put('stem', 'cp.resnet.conv1', 'cp.resnet.bn1', 'rgb')
        for li in (1, 2, 3, 4):
            for bi in (0, 1):
                p = 'cp.resnet.layer%d.%d' % (li, bi)
                put(p + '.c1', p + '.conv1', p + '.bn1', 'c3')
                put(p + '.c2', p + '.conv2', p + '.bn2', 'c3')
                if (P + p + '.downsample.0.weight') in sd:
                    put(p + '.ds', p + '.downsample.0', p + '.downsample.1', 'lin')
        for a in ('arm16', 'arm32'):
            put(a + '.conv', 'cp.%s.conv.conv' % a, 'cp.%s.conv.bn' % a, 'c3')
            put(a + '.att', 'cp.%s.conv_atten' % a, 'cp.%s.bn_atten' % a, 'lin')
        put('head32', 'cp.conv_head32.conv', 'cp.conv_head32.bn', 'up')
        put('head16', 'cp.conv_head16.conv', 'cp.conv_head16.bn', 'up')
        put('avg', 'cp.conv_avg.conv', 'cp.conv_avg.bn', 'lin')
        put('ffm.blk', 'ffm.convblk.conv', 'ffm.convblk.bn', 'lin')
        put('ffm.c1', 'ffm.conv1', None, 'lin')
        put('ffm.c2', 'ffm.conv2', None, 'lin')
        for o in ('conv_out', 'conv_out16', 'conv_out32'):
            put(o + '.conv', o + '.conv.conv', o + '.conv.bn', 'c3')
            put(o + '.out', o + '.conv_out', None, 'lin')

    def _pconv(self, x, key, cout, stride=1, **kw):
        Fr, H, W, _ = x.shape
        out = self._new(Fr, H // stride, W // stride, cout)
        return ops.conv(x, self.w['bn.' + key + '.weight'], cout, out, stride=stride, pad_lo=1,
                        bias=self.w.get('bn.' + key + '.bias'), **kw)

    def _plin(self, x, key, n, act=ops.ACT_NONE, out=None):
        if out is None:
            out = self._new(*x.shape[:-1], n)
        return ops.linear(x, self.w['bn.' + key + '.weight'], out, bias=self.w.get('bn.' + key + '.bias'), N=n, act=act)

    def _basic_block(self, x, p, cout, stride):
        """BasicBlock (`archs/pgtformer_arch.py:41-68`): relu(bn1(conv1)) -> bn2(conv2) ; relu(shortcut + residual)."""
        r = self._pconv(x, p + '.c1', cout, stride, act=ops.ACT_RELU)
        if ('bn.' + p + '.ds.weight') in self.w:
            Fr, H, W, cin = x.shape
            sc = self._new(Fr, H // stride, W // stride, cout)
            ops.conv(x, self.w['bn.' + p + '.ds.weight'], cout, sc, ksize=1, stride=stride, pad_lo=0,
                     bias=self.w['bn.' + p + '.ds.bias'])
        else:
            sc = x
        return self._pconv(r, p + '.c2', cout, 1, act=ops.ACT_RELU, residual=sc, relu_after_res=True)

    def parsing_net(self, x):
        """BiSeNet.forward (`archs/pgtformer_arch.py:365-379`) on the raw [F,3,H,W] image (ImageNet normalisation fused
        into the stem) -> conditioning map [F, H/16, W/16, 64] bf16 (57 channels used, zero padded)."""
        Fr, _, H, W = x.shape
        w = self.w
        # 7x7/2 stem on the tensor cores (im2col + ImageNet normalisation inside the kernel, folded BN + ReLU epilogue)
        t = ops.conv_rgb(x, w['bn.stem.weight'], w['bn.stem.bias'], self._new(Fr, H // 2, W // 2, 64), 7, 2, 3,
                         act=ops.ACT_RELU, mean3=(0.485, 0.456, 0.406), std3=(0.229, 0.224, 0.225))
        t = ops.maxpool3x3s2(t, self._new(Fr, H // 4, W // 4, 64))
        feats = []
        for li, cout, stride in ((1, 64, 1), (2, 128, 2), (3, 256, 2), (4, 512, 2)):
            t = self._basic_block(t, 'cp.resnet.layer%d.0' % li, cout, stride)
            t = self._basic_block(t, 'cp.resnet.layer%d.1' % li, cout, 1)
            feats.append(t)
        f8, f16, f32 = feats[1], feats[2], feats[3]
        # context path (:228-249)
        avg = self._plin(ops.global_avgpool(f32, self._new(Fr, 512)), 'avg', 128, act=ops.ACT_RELU)
        a32 = self._pconv(f32, 'arm32.conv', 128, act=ops.ACT_RELU)
        att = self._plin(ops.global_avgpool(a32, self._new(Fr, 128)), 'arm32.att', 128, act=ops.ACT_SIGMOID)
        s32 = ops.channel_affine(a32, att, self._new(*a32.shape), addv=avg)
        u32 = ops.conv_up2x(s32, w['bn.head32.weight'], 128, self._new(Fr, H // 16, W // 16, 128), bias=w['bn.head32.bias'],
                            act=ops.ACT_RELU)
        a16 = self._pconv(f16, 'arm16.conv', 128, act=ops.ACT_RELU)
        att = self._plin(ops.global_avgpool(a16, self._new(Fr, 128)), 'arm16.att', 128, act=ops.ACT_SIGMOID)
        s16 = ops.channel_affine(a16, att, self._new(*a16.shape), addm=u32)
        u16 = ops.conv_up2x(s16, w['bn.head16.weight'], 128, self._new(Fr, H // 8, W // 8, 128), bias=w['bn.head16.bias'],
                            act=ops.ACT_RELU)
        # feature fusion (:324-334)
        cat = self._new(Fr, H // 8, W // 8, 256)
        ops.copy2d(f8, cat[..., :128])
        ops.copy2d(u16, cat[..., 128:])
        fc = self._plin(cat, 'ffm.blk', 256, act=ops.ACT_RELU)
        at = self._plin(self._plin(ops.global_avgpool(fc, self._new(Fr, 256)), 'ffm.c1', 64, act=ops.ACT_RELU),
                        'ffm.c2', 256, act=ops.ACT_SIGMOID)
        fuse = ops.channel_affine(fc, at, self._new(*fc.shape), plus_one=True)
        # three 19-class heads (:147-150) -> bilinear(align_corners) to H/16 and concatenate
        o0 = self._plin(self._pconv(fuse, 'conv_out.conv', 256, act=ops.ACT_RELU), 'conv_out.out', 19,
                        out=self._new(Fr, H // 8, W // 8, 32))
        o1 = self._plin(self._pconv(u16, 'conv_out16.conv', 64, act=ops.ACT_RELU), 'conv_out16.out', 19,
                        out=self._new(Fr, H // 8, W // 8, 32))
        o2 = self._plin(self._pconv(u32, 'conv_out32.conv', 64, act=ops.ACT_RELU), 'conv_out32.out', 19,
                        out=self._new(Fr, H // 16, W // 16, 32))
        return ops.assemble_cond(o0, o1, o2, self._new(Fr, H // 16, W // 16, 64))

    # ------------------------------------------------------------------ encoder / decoder
    def encoder_frames(self, x):
        """The per-frame prefix of Encoder.forward (`archs/tdcrqvae3_arch.py:540-560`): conv_in and every level before
        the first one with attention, including the Downsample into it — nothing here looks across frames, so the
        streaming pipeline runs it once per distinct frame.  Returns (h, feats, next level)."""
        a = self.arch
        h = self.conv_in(x)
        feats = []
        lvl = 0
        while lvl < a.num_levels - 1 and not a.level_has_attn[lvl]:
            h = self._encoder_level(h, lvl, feats)
            lvl += 1
        return h, feats, lvl

    def conv_in(self, x, p='encoder.conv_in'):
        """encoder.conv_in on the fp32 NCHW frames.  Cin = 3: the kernel builds the patch rows itself; its epilogue also
        yields block 0's GroupNorm statistics."""
        a = self.arch
        Fr, _, H, W = x.shape
        h = self._new(Fr, H, W, a.ch)
        stats = None
        if self.fuse_gn_stats and (H * W) % 128 == 0 and a.ch == 64:
            tpf = H * W // 128
            stats = self._new(Fr * tpf * 4 * 64, dtype=torch.float32)
            h._pgt_gn = (stats, tpf * 4)
        ops.conv_rgb(x, self.w[p + '.weight'], self.w[p + '.bias'], h, 3, 1, 1, gn_stats=stats)
        return h

    def _encoder_level(self, h, lvl, feats):
        a = self.arch
        last = lvl == a.num_levels - 1
        Fr, H, W, _ = h.shape
        # a level whose output is an SFT skip tensor writes it into the [enc | dec | t] concat buffer of that fusion
        # (not the last level: its output carries GroupNorm statistics for mid.block_1 and must stay contiguous)
        slot = None
        if self.fuse_cat_in_place and self._fusing and lvl in a.fuse_level_key and not last:
            cat = self._cat_slot(Fr, H, W, a.level_ch[lvl])
            slot = cat[..., :a.level_ch[lvl]]
        for blk in range(a.num_res_blocks):
            # the next consumer of this level's output is a Normalize() only at the last level (mid.block_1);
            # otherwise it is the stride-2 Downsample conv, whose own epilogue feeds the next level's norm1
            nxt = last and blk == a.num_res_blocks - 1
            fin = slot if blk == a.num_res_blocks - 1 else None
            h = self.td_resblock(h, 'encoder.down.%d.block.%d' % (lvl, blk), a.level_ch[lvl],
                                 gn_next=nxt and not a.level_has_attn[lvl], out=None if a.level_has_attn[lvl] else fin)
            if a.level_has_attn[lvl]:
                h = self.encoder_layer(h, 'encoder.down.%d.attn.%d' % (lvl, blk), a.num_heads[lvl], a.depths[lvl],
                                       gn_next=nxt, out=fin)
        if slot is not None:
            h._pgt_cat = cat
        feats.append(h)
        if not last:
            h = self._conv3(h, 'encoder.down.%d.downsample.conv' % lvl, a.level_ch[lvl], stride=2, pad_lo=0, gn_out=True)
        return h

    def encoder_clips(self, h, feats, lvl):
        """The rest of Encoder.forward (`:560-573`) on clip-major frames."""
        a = self.arch
        while lvl < a.num_levels:
            h = self._encoder_level(h, lvl, feats)
            lvl += 1
        h = self.td_resblock(h, 'encoder.mid.block_1', a.level_ch[-1])
        h = self.encoder_layer(h, 'encoder.mid.attn_1', a.num_heads[-1], a.depths[-1], gn_next=True)
        h = self.td_resblock(h, 'encoder.mid.block_2', a.level_ch[-1], gn_next=True)
        zc = 2 * a.z_channels if a.double_z else a.z_channels
        return self._conv3(h, 'encoder.conv_out', zc, gn='encoder.norm_out'), feats

    def encoder(self, x):
        """Encoder.forward (`archs/tdcrqvae3_arch.py:540-573`); x fp32 NCHW -> (h [F,h,w,z], feats)."""
        h, feats, lvl = self.encoder_frames(x)
        return self.encoder_clips(h, feats, lvl)

    def _gather(self, t, idx):
        """t[idx] along the frame dimension, GroupNorm statistics included."""
        out = ops.gather_frames(t, idx, self._new(idx.numel(), *t.shape[1:], dtype=t.dtype))
        gn = getattr(t, '_pgt_gn', None)
        if gn is not None:
            st = gn[0].view(t.shape[0], -1)
            out._pgt_gn = (ops.gather_frames(st, idx, self._new(idx.numel(), st.shape[1], dtype=st.dtype)).view(-1), gn[1])
        return out

    def decoder(self, z, feats=None, wgt=0.0):
        """Decoder.forward (`archs/tdcrqvae3_arch.py:672-707`) / the inlined variant with SFT fusion
        (`archs/pgtformer_arch.py:680-710`).  z: [F,h,w,z_channels] bf16 -> out fp32 NCHW."""
        a = self.arch
        h = self._conv3(z, 'decoder.conv_in', a.level_ch[-1], gn_out=True)
        h = self.td_resblock(h, 'decoder.mid.block_1', a.level_ch[-1])
        h = self.encoder_layer(h, 'decoder.mid.attn_1', a.num_heads[-1], a.depths[-1], gn_next=True)
        h = self.td_resblock(h, 'decoder.mid.block_2', a.level_ch[-1], gn_next=True)
        for lvl in reversed(range(a.num_levels)):
            nblk = a.num_res_blocks + 1
            fuse = feats is not None and lvl in a.fuse_level_key and wgt > 0
            cat = getattr(feats[lvl], '_pgt_cat', None) if fuse else None
            for blk in range(nblk):
                # next consumer is a Normalize(): the next block of this level, or decoder.norm_out after the very
                # last block; after the level's last block comes the SFT concat / the upsample conv instead
                nxt = blk < nblk - 1 or (lvl == 0 and not fuse)
                C = a.level_ch[lvl]
                fin = cat[..., C:2 * C] if (cat is not None and blk == nblk - 1) else None
                h = self.td_resblock(h, 'decoder.up.%d.block.%d' % (lvl, blk), C,
                                     gn_next=nxt and not a.level_has_attn[lvl], out=None if a.level_has_attn[lvl] else fin)
                if a.level_has_attn[lvl]:
                    h = self.encoder_layer(h, 'decoder.up.%d.attn.%d' % (lvl, blk), a.num_heads[lvl], a.depths[lvl],
                                           gn_next=nxt, out=fin)
                if fin is not None:
                    h._pgt_cat = cat
            if fuse:
                h = self.fuse_sft(feats[lvl], h, a.fuse_level_key[lvl], wgt, gn_next=(lvl == 0))
            if lvl != 0:
                h = self.up2x(h, 'decoder.up.%d.upsample.conv' % lvl)
        return self.decoder_out(h)

    def up2x(self, h, p):
        """Upsample (nearest x2 + conv3x3) as four 2x2 phase convs; the epilogue emits the next norm1's statistics."""
        Fr, H, W, C = h.shape
        out = self._new(Fr, 2 * H, 2 * W, C)
        stats = None
        tpf = self._stats_tiles(H, W, C, 2, 1, 1)
        if self.fuse_gn_stats and tpf > 0 and C // 32 in (2, 4, 8, 16, 32):
            stats = self._new(Fr * 16 * tpf * 64, dtype=torch.float32)     # [frame][phase][tile][quadrant][32][2]
            out._pgt_gn = (stats, 16 * tpf)
        return ops.conv_up2x(h, self.w[p + '.weight'], C, out, bias=self.w[p + '.bias'], gn_stats=stats)

    def decoder_out(self, h, norm='decoder.norm_out', conv='decoder.conv_out', silu=True, out_ch=None):
        """norm (GroupNorm) + SiLU (unless silu=False) + conv -> fp32 NCHW [F, out_ch, H, W]."""
        out_ch = self.arch.out_ch if out_ch is None else out_ch
        Fr, H, W, _ = h.shape
        out = self._new(Fr, out_ch, H, W, dtype=torch.float32)
        if self.fuse_conv_out:
            # norm + SiLU + conv in one kernel: the normalised 512^2 tensor never reaches HBM
            st = getattr(h, '_pgt_gn', None)
            ab = ops.groupnorm_ab(h, self.w[norm + '.weight'], self.w[norm + '.bias'],
                                  self._new(Fr * 2 * h.shape[-1], dtype=torch.float32),
                                  stats=st[0] if st else None, chunks_per_frame=st[1] if st else 0)
            if ops.conv_out_gn(h, ab, self.w[conv + '.weight'], out_ch, self.w.get(conv + '.bias'), out,
                               silu=silu) is not None:
                return out
        self._conv3(h, conv, out_ch, out=out, gn=norm, gn_silu=silu, nchw=True)
        return out

    def parse_pos(self, x):
        """BiSeNet parsing features -> convpos 1x1 -> positional term [T, 512] bf16
        (`archs/pgtformer_arch.py:606-614`)."""
        Fr, _, H, W = x.shape
        cond = self.parsing_net(x)
        return self._lin(cond.view(Fr * (H // 16) * (W // 16), 64), 'convpos', 512, K=57)

    def global_transformer(self, lq, pos, clips):
        """feat_emb + 9 x TransformerSALayer + idx_pred_layer (`archs/pgtformer_arch.py:638-649`,
        `archs/codeformer_arch.py:121-137`) on [T, E] rows in natural (clip, frame, y, x) order;
        fp32 residual stream; returns fp32 logits [T, n_embed]."""
        a, wd = self.arch, self.w
        T, E = lq.shape[0], a.dim_embd
        L = T // clips
        q = self._lin(lq, 'feat_emb', E, out_dtype=torch.float32)
        for i in range(a.n_layers):
            p = 'ft_layers.%d' % i
            y, y2 = self._new(T, E), self._new(T, E)
            ops.layernorm(q, wd[p + '.norm1.weight'], wd[p + '.norm1.bias'], y, pos=pos, out2=y2)
            qk = self._lin(y2, p + '.self_attn.qk', 2 * E)
            v = self._lin(y, p + '.self_attn.v', E)
            att = ops.mha(qk[:, :E], qk[:, E:], v, clips, L, a.n_head, E // a.n_head, self._new(T, E))
            q = self._lin(att, p + '.self_attn.out_proj', E, out_dtype=torch.float32, residual=q)
            y = ops.layernorm(q, wd[p + '.norm2.weight'], wd[p + '.norm2.bias'], self._new(T, E))
            m = self._lin(y, p + '.linear1', 2 * E, act=ops.ACT_GELU)
            q = self._lin(m, p + '.linear2', E, out_dtype=torch.float32, residual=q)
        y = ops.layernorm(q, wd['idx_pred_layer.0.weight'], wd['idx_pred_layer.0.bias'], self._new(T, E))
        return self._lin(y, 'idx_pred_layer.1', self.depth * a.n_embed, out_dtype=torch.float32)

    # ------------------------------------------------------------------ full forwards
    @_on_device
    @torch.no_grad()
    def forward(self, x, w=1.0, adain=True, code_only=False, force_codes=None, frame_index=None):
        """PGTFormer.forward (`archs/pgtformer_arch.py:598-714`).  x: fp32 [b*3,3,H,W] in [0,1] on the
        device.  Returns (out, logits [b*3,h,w,D,K], lq_feat [b*3,h,w,E]) like the reference; force_codes [b*3,h,w,D].

        frame_index (streaming, `pgtformer_b200/video.py`): device int32 [b*3]; x then holds DISTINCT frames and
        clip frame f is x[frame_index[f]] — the per-frame work (BiSeNet, attention-free encoder levels) runs once per
        distinct frame and its results are gathered into clip order, bit-identical to running it per clip."""
        a = self.arch
        x = x.to(self.dev, torch.float32).contiguous()
        Fr, _, H, W = x.shape
        if frame_index is not None:
            Fr = frame_index.numel()
        if Fr % a.tf != 0 or H % 64 != 0 or W % 64 != 0:
            raise ValueError('expected b*3 frames with H, W multiples of 64, got %s' % (tuple(x.shape),))
        hh, ww = H // 16, W // 16
        T, E = Fr * hh * ww, a.dim_embd
        wd = self.w
        self._fusing = (not code_only) and float(w) > 0 and frame_index is None
        pos = self.parse_pos(x)
        # encoder
        if frame_index is None:
            h, feats = self.encoder(x)
        else:
            pos = self._gather(pos.view(x.shape[0], -1), frame_index).view(T, -1)
            h, feats, lvl = self.encoder_frames(x)
            # only the skip tensors the SFT fusion will read are worth moving (level 0 is 100 MB per clip and unused)
            feats = [self._gather(f, frame_index) if (i in a.fuse_level_key and w > 0) else f for i, f in enumerate(feats)]
            h, feats = self.encoder_clips(self._gather(h, frame_index), feats, lvl)
        h = h.view(T, -1)
        lq32 = self._lin(h, 'quant_conv', a.embed_dim, out_dtype=torch.float32)
        lq = self._lin(h, 'quant_conv', a.embed_dim)
        logits = self.global_transformer(lq, pos, Fr // 3)
        D = self.depth
        logits5 = logits.view(Fr, hh, ww, D, a.n_embed)
        lq_nhwc = lq32.view(Fr, hh, ww, a.embed_dim)
        if code_only:
            return logits5, lq_nhwc
        # quantise: argmax + codebook gather, AdaIN against lq, post_quant_conv
        codes = torch.empty(T * D, dtype=torch.int64, device=self.dev)
        quant = self._new(T, a.embed_dim, dtype=torch.float32)
        idx_in = force_codes.to(self.dev).reshape(T * D).contiguous() if force_codes is not None else None
        if D == 1:
            ops.argmax_gather(logits, wd['codebook'], codes, quant, idx_in=idx_in)
        else:
            # the [T, D*K] logits are [T*D, K] rows: one argmax per (token, depth), then the depth sum of the code rows
            if idx_in is None:
                ops.argmax_gather(logits.view(T * D, a.n_embed), wd['codebook'], codes, None)
            else:
                codes = idx_in
            ops.rq_embed(codes, 0, D - 1, wd['codebooks'], quant, ldi=D, ldd=1)
        self.last_codes = codes.view(Fr, hh, ww, D)
        if adain:
            quant = ops.adain(quant.view(Fr, hh * ww, -1), lq.view(Fr, hh * ww, -1), self._new(Fr, hh * ww, a.embed_dim))
        else:
            quant = quant.to(BF)
        z = self._lin(quant.reshape(T, a.embed_dim), 'post_quant_conv', a.z_channels)
        out = self.decoder(z.view(Fr, hh, ww, a.z_channels), feats, float(w))
        return out, logits5, lq_nhwc

    @_on_device
    @torch.no_grad()
    def forward_graphed(self, x, w=1.0, adain=True):
        """The same launch sequence replayed from a CUDA graph captured once per (shape, w, adain): removes the
        ~700 per-launch host costs (what bounds the reference's own b=1 sliding-window loop, `inference.py:47-74`).
        Returned tensors are the graph's static outputs: consume them before the next call."""
        x = x.to(self.dev, torch.float32).contiguous()
        key = (tuple(x.shape), float(w), bool(adain))
        if not hasattr(self, '_graphs'):
            self._graphs = {}
        entry = self._graphs.get(key)
        if entry is None:
            static_x = x.clone()
            side = torch.cuda.Stream(device=self.dev)
            side.wait_stream(torch.cuda.current_stream(self.dev))
            with torch.cuda.stream(side):                      # warm-up outside capture (lazy attribute / workspace setup)
                for _ in range(2):
                    self.forward(static_x, w=w, adain=adain)
            torch.cuda.current_stream(self.dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outs = self.forward(static_x, w=w, adain=adain)
            entry = (graph, static_x, outs)
            self._graphs[key] = entry
        graph, static_x, outs = entry
        static_x.copy_(x, non_blocking=True)
        graph.replay()
        return outs

    # ------------------------------------------------------------------ stage-I codec (TDCRQVAE3 methods)
    def _codebook(self, d=0):
        """fp32 codebook [K + 1, E] of depth d."""
        if d == 0 or self.arch.shared_codebook:
            return self.w['codebook']
        return self.w['codebooks'][d]

    def _codebook_pack(self, d=0):
        """bf16 copy + fp32 norms of depth d's codebook (l2_argmin_tc, soft_codes), once per load and distinct codebook."""
        key = 'codebook.pack' if d == 0 or self.arch.shared_codebook else 'codebook.pack.%d' % d
        if key not in self.w:
            self.w[key] = ops.codebook_pack(self._codebook(d), self.arch.n_embed)
        return self.w[key]

    def quantize(self, z):
        """RQBottleneck.quantize + compute_commitment_loss (`archs/tdcrqvae3_arch.py:294-352`) of z fp32 [T, E]:
        at each depth the exact L2 argmin of the residual over that depth's codebook, then residual -= e, aggregate
        += e in fp32.  Returns (codes int64 [T, D], z_q fp32 [T, E] = the aggregate of all depths, loss = mean over
        depths of mean((z - aggregate_d)^2))."""
        a = self.arch
        T, E = z.shape
        D = self.depth
        z_q = self._new(T, E, dtype=torch.float32)
        if D == 1:
            codes = torch.empty(T, dtype=torch.int64, device=self.dev)
            ops.l2_argmin_tc(z, self.w['codebook'], self._codebook_pack(), a.n_embed, codes, z_q)
            return codes.view(T, 1), z_q, (z - z_q).pow(2).mean()
        # codes depth-major, as l2_argmin_tc writes them; the residual is a scratch buffer (z itself is never copied)
        # and is updated after the argmin and its exhaustive fallback have both run
        codes = torch.empty(D, T, dtype=torch.int64, device=self.dev)
        r = self._new(T, E, dtype=torch.float32)
        losses = []
        for d in range(D):
            src = z if d == 0 else r
            ops.l2_argmin_tc(src, self._codebook(d), self._codebook_pack(d), a.n_embed, codes[d])
            ops.rq_residual(src, r if d < D - 1 else None, codes[d], self._codebook(d), z_q, d == 0)
            losses.append((z - z_q).pow(2).mean())
        return codes.t().contiguous(), z_q, torch.stack(losses).mean()

    @_on_device
    @torch.no_grad()
    def encode(self, x):
        """TDCRQVAE3.encode (`archs/tdcrqvae3_arch.py:774-777`): x fp32 [F,3,H,W] -> z_e fp32 NHWC [F,H/16,W/16,E]."""
        a = self.arch
        x = x.to(self.dev, torch.float32).contiguous()
        Fr, _, H, W = x.shape
        self._fusing = False                                   # the plain autoencoder has no SFT fusion
        h, _ = self.encoder(x)
        z_e = self._lin(h.view(Fr * (H // 16) * (W // 16), -1), 'quant_conv', a.embed_dim, out_dtype=torch.float32)
        return z_e.view(Fr, H // 16, W // 16, a.embed_dim)

    @_on_device
    @torch.no_grad()
    def decode(self, z_q):
        """TDCRQVAE3.decode (`:779-783`): z_q NHWC [F,h,w,E] -> post_quant_conv -> Decoder.forward (no SFT fusion)
        -> fp32 NCHW [F,3,16h,16w]."""
        a = self.arch
        Fr, hh, ww, E = z_q.shape
        self._fusing = False
        z = self._lin(z_q.to(self.dev, BF).reshape(Fr * hh * ww, E), 'post_quant_conv', a.z_channels)
        return self.decoder(z.view(Fr, hh, ww, a.z_channels))

    @_on_device
    @torch.no_grad()
    def embed_code(self, codes, d0=0, d1=None):
        """RQBottleneck.embed_code (`:355-368`): int64 codes [..., D] (each in [0, n_embed], the last row being the
        padding row; the gather does no range check) -> fp32 [T, E] = the sum of the code rows of depths d0 .. d1
        (default all: embed_code; d1 = j: the 'add' mode of embed_partial_code; d0 = d1 = j: its 'select' mode)."""
        self._fusing = False
        D = self.depth
        codes = codes.to(self.dev, torch.int64).reshape(-1, D).contiguous()
        d1 = D - 1 if d1 is None else d1
        quant = self._new(codes.shape[0], self.arch.embed_dim, dtype=torch.float32)
        if D == 1:
            ops.argmax_gather(None, self.w['codebook'], None, quant, idx_in=codes.view(-1))
        else:
            ops.rq_embed(codes, d0, d1, self.w['codebooks'], quant, ldi=D, ldd=1)
        return quant

    @_on_device
    @torch.no_grad()
    def embed_code_with_depth(self, codes):
        """RQBottleneck.embed_code_with_depth (`:371-391`): int64 codes [..., D] -> fp32 [T, D, E], one code row
        per depth (not summed)."""
        D = self.depth
        if D == 1:
            return self.embed_code(codes).unsqueeze(1)
        self._fusing = False
        codes = codes.to(self.dev, torch.int64).reshape(-1, D).contiguous()
        out = self._new(codes.shape[0], D, self.arch.embed_dim, dtype=torch.float32)
        for d in range(D):
            ops.rq_embed(codes, d, d, self.w['codebooks'], out[:, d], ldi=D, ldd=1)
        return out

    @_on_device
    @torch.no_grad()
    def soft_codes(self, z_e, temp, stochastic=False):
        """RQBottleneck.get_soft_codes (`:429-457`): z_e fp32 [T, E] -> (p fp32 [T, K], codes int64 [T]) at depth 1,
        (p fp32 [T, D, K], codes int64 [T, D]) at depth D.  Codes are the exact L2 argmin (== forward_vq's) or,
        stochastic, one draw per row from p with a seed taken on the device from the default CUDA generator
        (reproducible under torch.manual_seed, no host sync); each depth works on the residual the earlier codes left."""
        a = self.arch
        self._fusing = False
        z = z_e.to(self.dev, torch.float32).reshape(-1, a.embed_dim).contiguous()
        T = z.shape[0]
        if self.depth > 1:
            return self._soft_codes_rq(z, temp, stochastic)
        pack = self._codebook_pack()
        p = self._new(T, a.n_embed, dtype=torch.float32)
        ops.soft_codes(z, self.w['codebook'], pack[1], a.n_embed, temp, p)
        codes = torch.empty(T, dtype=torch.int64, device=self.dev)
        if stochastic:
            seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (2,), dtype=torch.int64, device=self.dev)
            ops.sample_codes(p, seed, codes)
        else:
            ops.l2_argmin_tc(z, self.w['codebook'], pack, a.n_embed, codes)
        return p, codes

    def _soft_codes_rq(self, z, temp, stochastic):
        a = self.arch
        T, D, K = z.shape[0], self.depth, a.n_embed
        p = self._new(T, D, K, dtype=torch.float32)
        codes = torch.empty(D, T, dtype=torch.int64, device=self.dev)
        r = self._new(T, a.embed_dim, dtype=torch.float32)
        for d in range(D):
            src = z if d == 0 else r
            pack = self._codebook_pack(d)
            ops.soft_codes_ld(src, self._codebook(d), pack[1], K, temp, p[:, d])
            if stochastic:
                seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (2,), dtype=torch.int64, device=self.dev)
                ops.sample_codes_ld(p[:, d], seed, codes[d])
            else:
                ops.l2_argmin_tc(src, self._codebook(d), pack, K, codes[d])
            if d < D - 1:
                ops.rq_residual(src, r, codes[d], self._codebook(d), None, d == 0)
        return p, codes.t().contiguous()

    @_on_device
    @torch.no_grad()
    def forward_vq(self, x, code_only=False):
        """TDCRQVAE3.forward (`archs/tdcrqvae3_arch.py:760-783`): encode -> residual quantiser -> decode."""
        a = self.arch
        z_e = self.encode(x)
        Fr, hh, ww, _ = z_e.shape
        T = Fr * hh * ww
        z_e = z_e.view(T, a.embed_dim)
        codes, z_q, loss = self.quantize(z_e)
        codes = codes.view(Fr, hh, ww, self.depth)
        z_q = z_q.view(Fr, hh, ww, -1)
        if code_only:
            return z_q, loss, codes
        return self.decode(z_q), loss, codes
