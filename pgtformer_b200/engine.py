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
import torch
import torch.nn.functional as F  # noqa: F401  (load-time weight padding only)

from . import degrade, ops
from .spec import Arch
from .swin3d import pack_blocks

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


def _fusing(feats, wgt):
    """Whether the SFT fusion blocks run: with skip tensors and a weight above 0 — or a device fp32 tensor of per-frame
    weights, which callers pass only for frames that all have w > 0 (a w = 0 frame skips the blocks, as the reference
    does, and the next GroupNorm then reads statistics of the unrounded res-block output, which the fused path does not
    reproduce)."""
    return feats is not None and (torch.is_tensor(wgt) or wgt > 0)


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
        """Every model's weights into kernel layouts by one rule.  The arch names the RGB stem, the upsample convs and
        the codebooks; any other 4-D weight is a 3x3 conv or a 1x1 conv (a linear), any other 2-D weight a linear, any
        1-D float tensor an fp32 vector.  The fused projections follow from the names present; the prefixes in
        arch.packed_apart are packed by a rule of their own."""
        a, sd, w = self.arch, self._sd, self.w
        names = [n for n in sd if not n.startswith(a.packed_apart)]
        for name in names:
            t = sd[name]
            if name == a.stem:
                w[name] = _pack_rgb(t.float())
            elif name in a.upsample_convs:
                w[name] = _pack_up2x(t.float())
            elif name.endswith('.weight') and t.dim() == 4:
                w[name] = _pack_conv(t.float()) if t.shape[2] == 3 else _pack_lin(t.float())
            elif name.endswith('.weight') and t.dim() == 2 and name not in a.codebooks:
                w[name] = _pack_lin(t.float())
            elif t.dtype.is_floating_point and t.dim() == 1:
                w[name] = t.float().contiguous()
        w['codebook'] = self._f32(a.codebooks[0])
        if self.depth > 1:
            # every distinct codebook stacked once [D or 1, K + 1, E], each zero-padded to the largest K + 1 rows: rq_embed
            # reads a shared one with depth stride 0, and depth d's padding row stays at index K_d
            cbs = [self._f32(k) for k in a.codebooks[:1 if a.shared_codebook else self.depth]]
            w['codebooks'] = torch.zeros(len(cbs), max(c.shape[0] for c in cbs), cbs[0].shape[1], dtype=torch.float32,
                                         device=self.dev)
            for d, cb in enumerate(cbs):
                w['codebooks'][d, :cb.shape[0]] = cb
        # Swin blocks: fused [q | k | v] projection and the expanded relative-position bias
        for name in names:
            if name.endswith('.attn.relative_position_bias_table'):
                p = name[:-len('.relative_position_bias_table')]
                heads = sd[name].shape[1]
                idx = sd[p + '.relative_position_index'].view(-1).long()
                w[p + '.bias_tab'] = sd[name].float()[idx].view(48, 48, heads).permute(2, 0, 1).contiguous()
                w[p + '.tab16'] = ops.window_tables(w[p + '.bias_tab'])     # wgmma window kernel: bias, 4 box layouts
                w[p + '.qkv.weight'] = _pack_lin(torch.cat([sd[p + '.q.weight'], sd[p + '.kv.weight']], 0).float())
                w[p + '.qkv.bias'] = torch.cat([sd[p + '.q.bias'], sd[p + '.kv.bias']], 0).float().contiguous()
                blk = p[:-len('.attn')]
                if sd[p + '.q.weight'].shape[1] == 256 and (blk + '.norm1.weight') in sd:
                    # norm1's affine folded into the projection the fused kernel applies to the normalised tile:
                    # (xh * g + b) W^T + c = xh (W * g)^T + (W b + c); products and sums in fp32, one bf16 rounding of W * g
                    wf = torch.cat([sd[p + '.q.weight'], sd[p + '.kv.weight']], 0)
                    wg, bg = fold_layernorm_affine(wf, w[p + '.qkv.bias'], sd[blk + '.norm1.weight'], sd[blk + '.norm1.bias'])
                    w[p + '.qkv_ln.weight'], w[p + '.qkv_ln.bias'] = _pack_lin(wg), bg
        # AttnBlock: q, k and v (1x1 convs of the same normalised input) as one [3C, C] projection
        for name in names:
            if name.endswith('.proj_out.weight'):
                p = name[:-len('.proj_out.weight')]
                w[p + '.qkv.weight'] = _pack_lin(torch.cat([sd[p + '.%s.weight' % n] for n in 'qkv'], 0).float())
                w[p + '.qkv.bias'] = torch.cat([sd[p + '.%s.bias' % n] for n in 'qkv'], 0).float().contiguous()
        # global transformer: in_proj split into the (q,k) projection of LN(x)+pos and the v projection of LN(x)
        for name in names:
            if name.endswith('.self_attn.in_proj_weight'):
                p = name[:-len('.in_proj_weight')]
                wi, bi = sd[name].float(), sd[p + '.in_proj_bias'].float()
                E = wi.shape[1]
                w[p + '.qk.weight'], w[p + '.qk.bias'] = _pack_lin(wi[:2 * E]), bi[:2 * E].contiguous()
                w[p + '.v.weight'], w[p + '.v.bias'] = _pack_lin(wi[2 * E:]), bi[2 * E:].contiguous()
        # Swin MLP halves: norm2's affine folded into fc1 (same algebra as norm1 -> q/kv above)
        for name in names:
            if name.endswith('.mlp.fc1.weight') and sd[name].shape == (256, 256):
                blk = name[:-len('.mlp.fc1.weight')]
                if (blk + '.norm2.weight') not in sd:
                    continue
                wg, bg = fold_layernorm_affine(sd[name], sd[blk + '.mlp.fc1.bias'], sd[blk + '.norm2.weight'],
                                               sd[blk + '.norm2.bias'])
                w[blk + '.mlp.fc1_ln.weight'], w[blk + '.mlp.fc1_ln.bias'] = _pack_lin(wg), bg
        # the prefixes packed by a rule of their own (BiSeNet, or one of TDRQVAE's Video-Swin BasicLayers), and
        # CodeFormer's learned positions
        self.swin = {}
        for prefix in a.packed_apart:
            if prefix == 'conditionnet.':
                self._repack_parsing()
            else:
                self.swin[prefix[:-1]] = pack_blocks(lambda k, p=prefix: sd.get(p + k), a.stages_atten)
        if 'position_emb' in sd:
            w['position_emb'] = sd['position_emb'].to(BF).contiguous()

    # ------------------------------------------------------------------ small helpers
    @property
    def depth(self):
        """Quantiser depth D = code_shape[2]: codes per token."""
        return int(self.arch.code_shape[2])

    def _new(self, *shape, dtype=BF):
        return torch.empty(*shape, dtype=dtype, device=self.dev)

    def _stats_tiles(self, H, W, cout, ksize, stride, pad_lo):
        """Tiles per frame of a conv whose epilogue emits the next GroupNorm's statistics; 0: no fused statistics.
        Fused statistics only where the conv's tile grid divides the frame: the models take frames of any multiple of
        64 (or 128), and at, say, 192 x 192 PGTFormer's level-0 Downsample (96 columns) gets 64-column tiles, whose
        last column of tiles would add rows past the frame's edge to the statistics (pgt_conv_tiles_exact)."""
        return ops.conv_tiles_exact(H, W, cout, ksize, stride, pad_lo)

    def _gn_stats(self, out, chunks_per_frame, into=None):
        """The next GroupNorm's statistics, filled by the epilogue that writes `out` (saves that GroupNorm a pass over
        the tensor): the fp32 buffer [frame][chunk][32 groups][2] (`into`, or a new one), attached as out._pgt_gn and
        returned for the producer's gn_stats.  None, with nothing attached, when out's channel count has no fused
        statistics, out is not contiguous or chunks_per_frame (32-row chunks per frame, 4 per 128-row tile) is 0."""
        if chunks_per_frame <= 0 or not ops.gn_stats_supported(out.shape[-1]) or not out.is_contiguous():
            return None
        stats = self._new(out.shape[0] * chunks_per_frame * 64, dtype=torch.float32) if into is None else into
        assert stats.numel() == out.shape[0] * chunks_per_frame * 64
        out._pgt_gn = (stats, chunks_per_frame)
        return stats

    def _gn(self, x, p, silu=True):
        gn = getattr(x, '_pgt_gn', None)
        if gn is not None:
            return ops.groupnorm_apply_stats(x, self.w[p + '.weight'], self.w[p + '.bias'], self._new(*x.shape), gn[0], gn[1],
                                             silu=silu)
        return ops.groupnorm_silu(x, self.w[p + '.weight'], self.w[p + '.bias'], self._new(*x.shape), silu=silu)

    def _conv3(self, x, p, cout, out=None, gn_out=False, gn=None, gn_silu=True, gn_into=None, **kw):
        """3x3 conv; gn: name of the Normalize() that precedes it, run as a separate pass: GroupNorm, then SiLU unless
        gn_silu=False (VQGAN's encoder tail).  gn_out: the epilogue also emits the next GroupNorm's statistics, into
        gn_into when given."""
        Fr, H, W, _ = x.shape
        stride = kw.get('stride', 1)
        if gn is not None:
            x = self._gn(x, gn, silu=gn_silu)
        if out is None:
            out = self._new(Fr, H // stride, W // stride, cout)
        stats = None
        if gn_out:
            stats = self._gn_stats(out, 4 * self._stats_tiles(H, W, cout, kw.get('ksize', 3), stride, kw.get('pad_lo', 1)),
                                   gn_into)
        return ops.conv(x, self.w[p + '.weight'], cout, out, bias=self.w.get(p + '.bias'), gn_stats=stats, **kw)

    def _lin(self, x, p, n, out=None, out_dtype=BF, gn_out=False, **kw):
        if out is None:
            out = self._new(*x.shape[:-1], n, dtype=out_dtype)
        stats = None
        if gn_out and out.dim() == 4 and out.dtype == BF and (out.shape[1] * out.shape[2]) % 128 == 0:
            stats = self._gn_stats(out, out.shape[1] * out.shape[2] // 32)
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
        if C == 256:
            # norm1 + the fused q/kv projection in one kernel (LN applied to the tile in shared memory; gamma / beta
            # already inside the weights, see _repack)
            qkv = ops.ln_linear(x, None, None, w[p + '.attn.qkv_ln.weight'], w[p + '.attn.qkv_ln.bias'],
                                self._new(Fr, H, W, 3 * C))
        else:
            y = ops.layernorm(x, w[p + '.norm1.weight'], w[p + '.norm1.bias'], self._new(Fr, H, W, C))
            qkv = self._lin(y, p + '.attn.qkv', 3 * C)
        a = self._new(Fr, H, W, C)
        if ops.window_attention_tc(qkv, Fr // 3, H, W, C, heads, shift, w[p + '.attn.tab16'], a) is None:
            ops.window_attention(qkv, Fr // 3, H, W, C, heads, shift, w[p + '.attn.bias_tab'], a)   # shapes the TMA kernel does not cover
        x = self._lin(a, p + '.attn.proj', C, residual=x)
        if C == 256:
            # norm2 + fc1 + GELU + fc2 + residual in one kernel (the hidden tile never leaves the SM; gamma / beta
            # already inside fc1, see _repack)
            out = self._new(Fr, H, W, C) if out is None else out
            stats = self._gn_stats(out, H * W // 32) if gn_next and (H * W) % 128 == 0 else None
            return ops.swin_mlp(x, None, None, w[p + '.mlp.fc1_ln.weight'], w[p + '.mlp.fc1_ln.bias'],
                                w[p + '.mlp.fc2.weight'], w[p + '.mlp.fc2.bias'], out, gn_stats=stats)
        y = ops.layernorm(x, w[p + '.norm2.weight'], w[p + '.norm2.bias'], self._new(Fr, H, W, C))
        m = self._lin(y, p + '.mlp.fc1', C, act=ops.ACT_GELU)
        return self._lin(m, p + '.mlp.fc2', C, residual=x, gn_out=gn_next, out=out)

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
        dec + w*(dec*scale + shift) is the epilogue of the last `shift` conv.  wgt: w, or a device fp32 [F] tensor of
        one w per frame of dec."""
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
        scale / shift branches -> dec + w*(dec*scale + shift) in the epilogue of the last `shift` conv (wgt: w, or a
        device fp32 [F] tensor of per-frame weights)."""
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
    def _walk(self, blocks, h, lo=0, hi=None, taps=None, outs=None, feats=None, wgt=0.0, gn_outs=None):
        """Runs blocks[lo:hi] of a block list (spec.Block entries) on h.  Returns (h, {taps[i]: output of block i}).
        outs {i: tensor}: block i (`res`, `swin` or `down`) writes its output there, a slice of an SFT concat buffer or a
        slot of a live ring (live_ring); gn_outs {i: fp32 buffer}: block i (`down`, the last of the frame blocks) writes
        the GroupNorm statistics it emits for the next block there.  A `fuse` block runs only with feats and wgt > 0 (or
        a device tensor of per-frame weights, see _fusing), on feats[its src].

        GroupNorm statistics: a block passes gn_next to its producer exactly when the next block that runs reads its
        input through a GroupNorm (`res`, `attn`, or the `norm` before conv_out); a `fuse` that does not run is not
        next.  Its epilogue then writes the statistics, and that GroupNorm skips its own pass over the tensor.  (The
        RGB conv_in and `up`, always followed by a `res`, always write them.)"""
        fusing = _fusing(feats, wgt)
        hi = len(blocks) if hi is None else hi
        outs, gn_outs, found = outs or {}, gn_outs or {}, {}
        for i in range(lo, hi):
            blk = blocks[i]
            kind, p, cout = blk.kind, blk.prefix, blk.cout
            if kind == 'fuse' and not fusing:
                continue
            nxt = next((b.kind in ('res', 'attn', 'norm') for b in blocks[i + 1:] if fusing or b.kind != 'fuse'), False)
            if kind == 'conv_in':
                h = self.conv_in(h, p) if p + '.weight' == self.arch.stem else self._conv3(h, p, cout, gn_out=nxt)
            elif kind == 'res':
                h = self.td_resblock(h, p, cout, gn_next=nxt, out=outs.get(i), shortcut=self.arch.res_shortcut)
            elif kind == 'attn':
                h = self.attn_block(h, p, gn_next=nxt)
            elif kind == 'swin':
                h = self.encoder_layer(h, p, blk.heads, blk.depth, gn_next=nxt, out=outs.get(i))
            elif kind == 'down':
                h = self._conv3(h, p + '.conv', cout, stride=2, pad_lo=0, gn_out=nxt, out=outs.get(i),
                                gn_into=gn_outs.get(i))
            elif kind == 'up':
                h = self.up2x(h, p + '.conv')
            elif kind == 'fuse':
                h = self.fuse_sft(feats[blk.src], h, p[len('fuse_convs_dict.'):], wgt, gn_next=nxt)
            else:
                raise AssertionError(kind)
            if taps and i in taps:
                found[taps[i]] = h
        return h, found

    @staticmethod
    def _cat_half(cat, lo, C):
        """cat[..., lo:lo + C] of an SFT concat buffer, marked as its slice so that fuse_sft reads it in place."""
        half = cat[..., lo:lo + C]
        half._pgt_cat = cat
        return half

    def encoder_frames(self, x, outs=None, gn_outs=None):
        """The per-frame prefix of Encoder.forward (`archs/tdcrqvae3_arch.py:540-560`): conv_in and every level before
        the first one with attention, including the Downsample into it — nothing here looks across frames, so the
        streaming pipeline runs it once per distinct frame.  Returns (h, {level: output}, index of the next block)."""
        a = self.arch
        h, feats = self._walk(a.enc_blocks, x, 0, a.frame_blocks, a.enc_taps, outs, gn_outs=gn_outs)
        return h, feats, a.frame_blocks

    def conv_in(self, x, p='encoder.conv_in'):
        """encoder.conv_in on the fp32 NCHW frames.  Cin = 3: the kernel builds the patch rows itself; its epilogue also
        yields block 0's GroupNorm statistics (a.ch = 64 or 128)."""
        a = self.arch
        Fr, _, H, W = x.shape
        h = self._new(Fr, H, W, a.ch)
        stats = self._gn_stats(h, H * W // 32) if (H * W) % 128 == 0 and a.ch in (64, 128) else None
        ops.conv_rgb(x, self.w[p + '.weight'], self.w[p + '.bias'], h, 3, 1, 1, gn_stats=stats)
        return h

    def encoder_clips(self, h, feats, i, outs=None):
        """The rest of Encoder.forward (`:560-573`) on clip-major frames, from block i; feats: the level outputs so
        far.  Returns (h [F,h,w,z], the output of every level)."""
        a = self.arch
        h, more = self._walk(a.enc_blocks, h, i, len(a.enc_blocks) - 2, a.enc_taps, outs)
        norm, conv = a.enc_blocks[-2:]
        return self._conv3(h, conv.prefix, conv.cout, gn=norm.prefix), list(feats.values()) + list(more.values())

    def encoder(self, x, fusing=False):
        """Encoder.forward (`archs/tdcrqvae3_arch.py:540-573`); x fp32 NCHW -> (h [F,h,w,z], feats).  fusing: the SFT
        fusion will read the level outputs, so each one (but the last level's, which carries GroupNorm statistics for
        mid.block_1 and must stay contiguous) is written straight into the encoder half of its concat buffer."""
        a = self.arch
        outs = {}
        if fusing:
            Fr, _, H, W = x.shape
            for i, lvl in a.enc_taps.items():
                C = a.level_ch[lvl]
                if lvl in a.fuse_level_key and lvl != a.num_levels - 1:
                    outs[i] = self._cat_half(self._cat_slot(Fr, H >> lvl, W >> lvl, C), 0, C)
        return self.encoder_clips(*self.encoder_frames(x, outs), outs)

    def _gather(self, t, idx):
        """t[idx] along the frame dimension."""
        return ops.gather_frames(t, idx, self._new(idx.numel(), *t.shape[1:], dtype=t.dtype))

    def decoder(self, z, feats=None, wgt=0.0):
        """Decoder.forward (`archs/tdcrqvae3_arch.py:672-707`) / the inlined variant with SFT fusion
        (`archs/pgtformer_arch.py:680-710`), or VQGAN's Generator.forward (`archs/vqgan_arch.py:337-341`) / with
        CodeFormer's fusion (`archs/codeformer_arch.py:356-363`).  z: [F,h,w,C] bf16 -> out fp32 NCHW.  A level whose
        encoder output sits in an SFT concat buffer writes its own output into the decoder half.  wgt: w, or a device
        fp32 [F] tensor of per-frame weights (_fusing)."""
        blocks = self.arch.dec_blocks
        outs = {}
        for i, b in enumerate(blocks):
            cat = getattr(feats[b.src], '_pgt_cat', None) if b.kind == 'fuse' and _fusing(feats, wgt) else None
            if cat is not None:
                outs[i - 1] = self._cat_half(cat, b.cout, b.cout)
        h, _ = self._walk(blocks, z, 0, len(blocks) - 2, outs=outs, feats=feats, wgt=wgt)
        norm, conv = blocks[-2:]
        return self.decoder_out(h, norm.prefix, conv.prefix, conv.cout, self.arch.dec_tail_silu)

    def up2x(self, h, p):
        """Upsample (nearest x2 + conv3x3) as four 2x2 phase convs; the epilogue emits the next norm1's statistics."""
        Fr, H, W, C = h.shape
        out = self._new(Fr, 2 * H, 2 * W, C)
        stats = self._gn_stats(out, 16 * self._stats_tiles(H, W, C, 2, 1, 1))     # [frame][phase][tile][quadrant]
        return ops.conv_up2x(h, self.w[p + '.weight'], C, out, bias=self.w[p + '.bias'], gn_stats=stats)

    def decoder_out(self, h, norm, conv, out_ch, silu):
        """norm (GroupNorm) + SiLU (unless silu=False) + conv -> fp32 NCHW [F, out_ch, H, W]."""
        Fr, H, W, _ = h.shape
        out = self._new(Fr, out_ch, H, W, dtype=torch.float32)
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

    def parse_pos(self, x, out=None):
        """BiSeNet parsing features -> convpos 1x1 -> positional term [T, 512] bf16
        (`archs/pgtformer_arch.py:606-614`), written into out when given."""
        Fr, _, H, W = x.shape
        cond = self.parsing_net(x)
        return self._lin(cond.view(Fr * (H // 16) * (W // 16), 64), 'convpos', 512, K=57, out=out)

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
        if frame_index is not None:
            return self._window_tail(self._frame_pass(x, w), frame_index, w, adain, code_only, force_codes)
        pos = self.parse_pos(x)
        h, feats = self.encoder(x, fusing=not code_only and float(w) > 0)
        return self._restore(h, feats, pos, w, adain, code_only, force_codes)

    def _frame_pass(self, x, w=0.0, ring=None, slot=0):
        """The per-frame work — parse_pos and encoder_frames — of distinct fp32 frames x [n,3,H,W], as their per-frame
        record: {'pos': convpos rows [n, T/n, 512], 'h': the frame blocks' output [n, ...], 'h_stats': the GroupNorm
        statistics [n, chunks * 64] h's producer writes for the next block (when it writes any), 'feats': {level:
        [n, ...]}, for w > 0 the skip tensors of the per-frame levels the SFT fusion reads (the others are never moved:
        level 0 is 100 MB per clip and unused)}.  With ring (live_ring: the record of a ring's rows) the producers write
        the n frames straight into rows slot .. slot + n - 1 of ring, and the levels kept are those the ring has room
        for."""
        a = self.arch
        last, n = a.frame_blocks - 1, x.shape[0]
        outs, gn_outs = {}, {}
        if ring is None:
            levels = list(a.fuse_level_key) if float(w) > 0 else []
        else:
            rows = slice(slot, slot + n)
            levels = list(ring['feats'])
            outs = {i: ring['feats'][lvl][rows] for i, lvl in a.enc_taps.items() if lvl in levels}
            outs[last] = ring['h'][rows]
            if 'h_stats' in ring:
                gn_outs[last] = ring['h_stats'][rows].view(-1)
        pos = self.parse_pos(x, out=None if ring is None else ring['pos'][rows].flatten(0, 1))
        h, feats, _ = self.encoder_frames(x, outs, gn_outs)
        rec = {'pos': pos.view(n, -1, pos.shape[-1]), 'h': h,
               'feats': {lvl: f for lvl, f in feats.items() if lvl in levels}}
        gn = getattr(h, '_pgt_gn', None)
        if gn is not None:
            rec['h_stats'] = gn[0].view(n, -1)
        return rec

    def _window_tail(self, rec, index, w, adain, code_only=False, force_codes=None):
        """forward from a per-frame record (_frame_pass, live_ring) on: its entries gathered into clip order by the
        device int32 window index [b*3] (pgt_gather_frames), h's GroupNorm statistics beside h, then encoder_clips and
        _restore, whose result it returns.  The skip tensors are gathered only when the fusion runs (_fusing)."""
        a = self.arch
        pos = self._gather(rec['pos'], index)
        fusing = _fusing(rec['feats'], w)
        feats = {lvl: self._gather(rec['feats'][lvl], index) if fusing and lvl in rec['feats'] else None
                 for i, lvl in a.enc_taps.items() if i < a.frame_blocks}
        h = self._gather(rec['h'], index)
        if 'h_stats' in rec:
            h._pgt_gn = (self._gather(rec['h_stats'], index).view(-1), rec['h_stats'].shape[1] // 64)
        h, feats = self.encoder_clips(h, feats, a.frame_blocks)
        return self._restore(h, feats, pos.view(-1, pos.shape[-1]), w, adain, code_only, force_codes)

    def _restore(self, h, feats, pos, w, adain, code_only=False, force_codes=None):
        """forward from the encoder's output h [F,h,w,C] on: quant_conv -> global transformer -> argmax (or
        force_codes) / AdaIN -> post_quant_conv -> decoder with SFT fusion of feats.  Per frame (the live pool's
        batches of streams with their own settings): w may be a device fp32 [F] tensor of weights, all > 0 (_fusing),
        and adain a device int32 [F] tensor of flags (pgt_adain_frames: AdaIN where set, a bf16 rounding elsewhere)."""
        a = self.arch
        Fr, hh, ww, _ = h.shape
        T = Fr * hh * ww
        wd = self.w
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
        if torch.is_tensor(adain):
            quant = ops.adain(quant.view(Fr, hh * ww, -1), lq.view(Fr, hh * ww, -1), self._new(Fr, hh * ww, a.embed_dim),
                              flags=adain)
        elif adain:
            quant = ops.adain(quant.view(Fr, hh * ww, -1), lq.view(Fr, hh * ww, -1), self._new(Fr, hh * ww, a.embed_dim))
        else:
            quant = quant.to(BF)
        z = self._lin(quant.reshape(T, a.embed_dim), 'post_quant_conv', a.z_channels)
        out = self.decoder(z.view(Fr, hh, ww, a.z_channels), feats, w if torch.is_tensor(w) else float(w))
        return out, logits5, lq_nhwc

    @_on_device
    @torch.no_grad()
    def graphed(self, method, tensors, writes=(), **scalars):
        """method(*tensors, **scalars) replayed from a CUDA graph: removes the host cost of every launch (Python, ctypes,
        the output allocations and tensor-map lookups), up to a third of a call at b = 1 (DESIGN §6c).

        One graph per key = (method, shapes and dtypes of the tensors, scalars), kept by this engine: a new key runs the
        method twice on a side stream (the lazy one-time set-up: kernel attributes, constant tables, codebook packs,
        workspaces) and then captures it on this engine's capture stream (on its device), into a memory pool of its own;
        scratch taken during the capture comes from that pool (ops._gn_workspace).  Every call copies the tensors into the graph's
        static inputs and replays it; tensors at the indices in `writes` are ones the method updates in place, copied
        back after the replay.  Returns the graph's static outputs: consume them before the next call.  Arguments are
        checked by the caller before this: a capture never starts on an argument the method would reject, and a key
        whose warm-up raises stores nothing.

        A graph here is a pure function of its inputs.  The live steps (video.LivePool, pool_step), whose ring of
        per-frame results persists across replays, are captured by their pool through _capture too, all in one memory
        pool: one graph per (new frames, windows) count, reading its slot and window indices from device buffers the
        pool fills before each replay."""
        tensors = [t.to(self.dev) for t in tensors]
        key = (method.__name__, tuple((tuple(t.shape), t.dtype) for t in tensors), tuple(sorted(scalars.items())))
        if not hasattr(self, '_graphs'):
            self._graphs = {}
        entry = self._graphs.get(key)
        if entry is None:
            static = [torch.empty(t.shape, dtype=t.dtype, device=self.dev) for t in tensors]
            for s, t in zip(static, tensors):
                s.copy_(t)
            entry = self._graphs[key] = (static,) + self._capture(lambda: method(*static, **scalars))
        static, graph, outs = entry
        for s, t in zip(static, tensors):
            s.copy_(t, non_blocking=True)
        graph.replay()
        for i in writes:
            tensors[i].copy_(static[i], non_blocking=True)
        return outs

    def _capture(self, run, pool=None):
        """(graph, what run() returned in it): run() twice on a side stream (the lazy one-time set-up: kernel
        attributes, constant tables, codebook packs, workspaces), then captured as a CUDA graph on this engine's
        capture stream, on its device, into `pool` (None: a memory pool of the graph's own)."""
        if not hasattr(self, 'capture_stream'):
            self.capture_stream = torch.cuda.Stream(device=self.dev)
        cur = torch.cuda.current_stream(self.dev)
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(cur)
        try:
            with torch.cuda.stream(side):
                for _ in range(2):
                    run()
        finally:
            cur.wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=pool, stream=self.capture_stream):
            out = run()
        return graph, out

    def forward_graphed(self, x, w=1.0, adain=True):
        """forward replayed from a CUDA graph captured once per (shape, w, adain) (graphed): removes the ~700
        per-launch host costs (what bounds the reference's own b=1 sliding-window loop, `inference.py:47-74`).
        Returned tensors are the graph's static outputs: consume them before the next call."""
        x = x.to(self.dev, torch.float32).contiguous()
        return self.graphed(self.forward, (x,), w=float(w), adain=bool(adain))

    # ------------------------------------------------------------------ video: batched windows and the live ring
    @_on_device
    @torch.no_grad()
    def restore_windows(self, frames_u8, index, w=1.0, adain=True, reuse_frames=True, size=None, downscale=None):
        """One batch of VideoRestorer: rgb24 frames [Fd,H,W,3] uint8 on the device and the device int32 window index
        [3n] into them -> the restored middle frames, rgb24 [n,H,W,3] uint8 on the device.  size = (H, W): the frames
        are [Fd,h,w,3] sources of any size, upsampled to H x W as the reference's test set does
        (ops.u8hwc_resize_to_f32nchw).  downscale (with size): the frames are ground truth, degraded as the test set's
        `lr` protocol does, basicsr's imresize by that scale into fp32 (degrade.resize), then bilinear to H x W
        (ops.f32nchw_resize_to_f32nchw); the caller has checked the scale against the frames (degrade.plan)."""
        Fd, h, w_src, _ = frames_u8.shape
        if downscale is not None:
            H, W = size
            lo = degrade.resize(frames_u8, downscale, self._new(Fd, 3, *degrade.out_size((h, w_src), downscale),
                                                                dtype=torch.float32))
            x = ops.f32nchw_resize_to_f32nchw(lo, self._new(Fd, 3, H, W, dtype=torch.float32))
        elif size is None:
            H, W = h, w_src
            x = ops.u8hwc_to_f32nchw(frames_u8, self._new(Fd, 3, H, W, dtype=torch.float32))
        else:
            H, W = size
            x = ops.u8hwc_resize_to_f32nchw(frames_u8, self._new(Fd, 3, H, W, dtype=torch.float32), (h, w_src))
        if reuse_frames:
            out = self.forward(x, w=w, adain=adain, frame_index=index)[0]
        else:
            xc = ops.gather_frames(x, index, self._new(index.numel(), 3, H, W, dtype=torch.float32))
            out = self.forward(xc, w=w, adain=adain)[0]
        n = index.numel() // 3
        return ops.f32nchw_to_u8hwc(out, torch.empty(n, H, W, 3, dtype=torch.uint8, device=self.dev), first=1, step=3)

    @_on_device
    @torch.no_grad()
    def restore_and_score(self, frames_u8, index, gt_u8, w=1.0, adain=True, reuse_frames=True, size=None,
                          downscale=None):
        """restore_windows, then the restored frames scored against gt_u8 (rgb24 [n,H,W,3] uint8 on the device) before
        they leave it (ops.frame_scores) -> (restored, sse int64 [n], per-channel ssim fp64 [n,3])."""
        out = self.restore_windows(frames_u8, index, w=w, adain=adain, reuse_frames=reuse_frames, size=size,
                                   downscale=downscale)
        return (out,) + ops.frame_scores(out, gt_u8)

    @_on_device
    @torch.no_grad()
    def live_ring(self, H, W, w, streams=1):
        """The per-frame record (_frame_pass) of 4 * streams rows, for frame_step / window_step / pool_step: row
        3 s + (j mod 3) holds frame j of stream s, and rows 3 * streams + k are the staging rows pool_step's new frames
        are computed into.  Allocated here, outside any graph's memory pool, so that graphs captured later can all
        write and read the same addresses.  Shapes are those of one run of the per-frame work."""
        if H % 64 or W % 64:
            raise ValueError('expected H, W multiples of 64, got %dx%d' % (H, W))
        rows = 4 * int(streams)
        rec = self._frame_pass(torch.zeros(1, 3, H, W, dtype=torch.float32, device=self.dev), w)
        ring = {k: self._new(rows, *t.shape[1:], dtype=t.dtype) for k, t in rec.items() if k != 'feats'}
        ring['feats'] = {lvl: self._new(rows, *f.shape[1:], dtype=f.dtype) for lvl, f in rec['feats'].items()}
        return ring

    @staticmethod
    def ring_entries(ring):
        """Every tensor of a live ring (live_ring), one row per frame: pos, h, h_stats when present, the kept feats."""
        return [ring[k] for k in ('pos', 'h', 'h_stats') if k in ring] + list(ring['feats'].values())

    @_on_device
    @torch.no_grad()
    def frame_step(self, x, slot, ring):
        """The per-frame work of fp32 frames x [B,3,H,W] — parse_pos and encoder_frames — written into rows
        slot .. slot + B - 1 of ring (live_ring) by the producing kernels themselves."""
        self._frame_pass(x, ring=ring, slot=slot)

    @_on_device
    @torch.no_grad()
    def window_step(self, index, w, adain, ring, out_u8):
        """The windows (f[i-1], f[i], f[i+1]) restored from the ring rows of index (device int32 [3 Bw]), exactly as
        forward(frame_index=index) computes them.  Writes the middle frames into out_u8 (rgb24 [Bw,H,W,3] uint8).  w and
        adain: scalars, or device tensors of one value per frame of index (_restore)."""
        out = self._window_tail(ring, index, w, adain)[0]
        return ops.f32nchw_to_u8hwc(out, out_u8, first=1, step=3)

    @_on_device
    @torch.no_grad()
    def pool_step(self, u8, x, ring, slots, index, w, adain, out_u8, sizes=None):
        """One step of a pool of live streams (video.LivePool) on a live_ring of S streams and its rgb24 frames u8
        [4S,H,W,3] (the same rows).  The B = slots.numel() new frames, already in u8's staging rows 3S .. 3S + B - 1,
        go to fp32 in x [>=B,3,H,W] and through frame_step into the ring's staging rows; every ring entry and the rgb24
        frame are then scattered to the frames' slots (slots: device int32 [B]; h's GroupNorm statistics travel as
        their own entry).  Then the windows of index (device int32 [3 Bw], ring rows; None for none) are restored into
        out_u8 [Bw,H,W,3], with w and adain as window_step takes them.  sizes (device int32 [B, 3]): the staging rows
        hold source frames of (h, w) at a byte offset from row 3S, each upsampled to H x W
        (ops.u8hwc_resize_to_f32nchw); None: frames at H x W.  Nothing else is touched, so a step replays from a CUDA
        graph given its index tensors (and its per-frame settings and source sizes)."""
        if slots is not None:
            B, st = slots.numel(), u8.shape[0] // 4 * 3
            if sizes is None:
                xs = ops.u8hwc_to_f32nchw(u8[st:st + B], x[:B])
            else:
                xs = ops.u8hwc_resize_to_f32nchw(u8[st:st + B], x[:B], tuple(u8.shape[1:3]), sizes)
            self.frame_step(xs, st, ring)
            for t in self.ring_entries(ring) + [u8]:
                ops.scatter_frames(t[st:st + B], slots, t)
        if index is not None:
            self.window_step(index, w, adain, ring, out_u8)

    # ------------------------------------------------------------------ stage-I codec (TDCRQVAE3 methods)
    def _codebook(self, d=0):
        """fp32 codebook [K + 1, E] of depth d."""
        if d == 0 or self.arch.shared_codebook:
            return self.w['codebook']
        return self.w['codebooks'][d]

    def _n_embed(self, d=0):
        """Codes in depth d's codebook (the rows before its padding row): arch.n_embeds[d] for the RQ archs, which list
        one size per depth; an arch with one codebook size and no such list (VQGAN's, a bare quantiser's) has n_embed."""
        a = self.arch
        return a.n_embeds[d] if hasattr(a, 'n_embeds') else a.n_embed

    def _codebook_pack(self, d=0):
        """bf16 copy + fp32 norms of depth d's codebook (l2_argmin_tc, soft_codes), once per load and distinct codebook."""
        key = 'codebook.pack' if d == 0 or self.arch.shared_codebook else 'codebook.pack.%d' % d
        if key not in self.w:
            self.w[key] = ops.codebook_pack(self._codebook(d), self._n_embed(d))
        return self.w[key]

    def _argmin(self, *a, **k):
        """The exact L2 argmin quantize runs (RQVAEEngine: the codebook-split one)."""
        return ops.l2_argmin_tc(*a, **k)

    def quantize(self, z):
        """RQBottleneck.quantize + compute_commitment_loss (`archs/tdcrqvae3_arch.py:294-352`) of z fp32 [T, E]:
        at each depth the exact L2 argmin of the residual over that depth's codebook, then residual -= e, aggregate
        += e in fp32.  Returns (codes int64 [T, D], z_q fp32 [T, E] = the aggregate of all depths, loss = mean over
        depths of mean((z - aggregate_d)^2))."""
        T, E = z.shape
        D = self.depth
        z_q = self._new(T, E, dtype=torch.float32)
        if D == 1:
            codes = torch.empty(T, dtype=torch.int64, device=self.dev)
            self._argmin(z, self.w['codebook'], self._codebook_pack(), self._n_embed(0), codes, z_q)
            return codes.view(T, 1), z_q, (z - z_q).pow(2).mean()
        # codes depth-major, as l2_argmin_tc writes them; the residual is a scratch buffer (z itself is never copied)
        # and is updated after the argmin and its exhaustive fallback have both run
        codes = torch.empty(D, T, dtype=torch.int64, device=self.dev)
        r = self._new(T, E, dtype=torch.float32)
        losses = []
        for d in range(D):
            src = z if d == 0 else r
            self._argmin(src, self._codebook(d), self._codebook_pack(d), self._n_embed(d), codes[d])
            ops.rq_residual(src, r if d < D - 1 else None, codes[d], self._codebook(d), z_q, d == 0)
            losses.append((z - z_q).pow(2).mean())
        return codes.t().contiguous(), z_q, torch.stack(losses).mean()

    @_on_device
    @torch.no_grad()
    def encode(self, x):
        """TDCRQVAE3.encode (`archs/tdcrqvae3_arch.py:774-777`): x fp32 [F,3,H,W] -> z_e fp32 NHWC [F,h,w,E], h x w the
        encoder's latent map (H/16 x W/16 for the four-downsample encoders)."""
        a = self.arch
        x = x.to(self.dev, torch.float32).contiguous()
        h, _ = self.encoder(x)
        Fr, hh, ww, _ = h.shape
        z_e = self._lin(h.view(Fr * hh * ww, -1), 'quant_conv', a.embed_dim, out_dtype=torch.float32)
        return z_e.view(Fr, hh, ww, a.embed_dim)

    @_on_device
    @torch.no_grad()
    def decode(self, z_q):
        """TDCRQVAE3.decode (`:779-783`): z_q NHWC [F,h,w,E] -> post_quant_conv -> Decoder.forward (no SFT fusion)
        -> fp32 NCHW [F,3,16h,16w]."""
        a = self.arch
        Fr, hh, ww, E = z_q.shape
        z = self._lin(z_q.to(self.dev, BF).reshape(Fr * hh * ww, E), 'post_quant_conv', a.z_channels)
        return self.decoder(z.view(Fr, hh, ww, a.z_channels))

    @_on_device
    @torch.no_grad()
    def embed_code(self, codes, d0=0, d1=None):
        """RQBottleneck.embed_code (`:355-368`): int64 codes [..., D] (each in [0, n_embed], the last row being the
        padding row; the gather does no range check) -> fp32 [T, E] = the sum of the code rows of depths d0 .. d1
        (default all: embed_code; d1 = j: the 'add' mode of embed_partial_code; d0 = d1 = j: its 'select' mode)."""
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
    def decode_code(self, codes):
        """decode of embed_code: int64 codes [F, h, w, D] -> the depth sum of their code rows, decoded to fp32 NCHW."""
        Fr, hh, ww, _ = codes.shape
        return self.decode(self.embed_code(codes).view(Fr, hh, ww, self.arch.embed_dim))

    @_on_device
    @torch.no_grad()
    def embed_code_with_depth(self, codes):
        """RQBottleneck.embed_code_with_depth (`:371-391`): int64 codes [..., D] -> fp32 [T, D, E], one code row
        per depth (not summed)."""
        D = self.depth
        if D == 1:
            return self.embed_code(codes).unsqueeze(1)
        codes = codes.to(self.dev, torch.int64).reshape(-1, D).contiguous()
        out = self._new(codes.shape[0], D, self.arch.embed_dim, dtype=torch.float32)
        for d in range(D):
            ops.rq_embed(codes, d, d, self.w['codebooks'], out[:, d], ldi=D, ldd=1)
        return out

    @_on_device
    @torch.no_grad()
    def soft_codes(self, z_e, temp, stochastic=False):
        """RQBottleneck.get_soft_codes (`:429-457`): z_e fp32 [T, E] -> (p fp32 [T, D, K], codes int64 [T, D]).  Codes
        are the exact L2 argmin (== forward_vq's) or, stochastic, one draw per row from p with a seed taken on the device
        from the default CUDA generator (reproducible under torch.manual_seed, no host sync); each depth works on the
        residual the earlier codes left and writes K-slice d of p."""
        a = self.arch
        z = z_e.to(self.dev, torch.float32).reshape(-1, a.embed_dim).contiguous()
        T, D, K = z.shape[0], self.depth, a.n_embed
        p = self._new(T, D, K, dtype=torch.float32)
        codes = torch.empty(D, T, dtype=torch.int64, device=self.dev)
        r = self._new(T, a.embed_dim, dtype=torch.float32) if D > 1 else None
        for d in range(D):
            src = z if d == 0 else r
            pack = self._codebook_pack(d)
            ops.soft_codes(src, self._codebook(d), pack[1], K, temp, p[:, d])
            if stochastic:
                seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (2,), dtype=torch.int64, device=self.dev)
                ops.sample_codes(p[:, d], seed, codes[d])
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
