"""H100 launch sequence of TDRQVAE (`archs/tdrqvae_arch.py:787-976`): the 2-D RQ-VAE Encoder / Decoder with dense
AttnBlocks, the depth-1 L2-argmin quantiser and the two Video-Swin BasicLayers around it, over libpgt_b200.so.

Layout as in engine.py: channels-last bf16 feature maps [F = b*t, H, W, C], frames of a clip contiguous.  The
quant_conv output rows are therefore already in (b, t, y, x) order, the 'b d h w c' token order of the Video-Swin
layers, so the reference's permutes around tdswin_pre / tdswin_post are never materialised.  Every op is a call into
the C ABI; there is no PyTorch / CPU fallback."""
import torch

from . import ops
from .engine import BF, Engine, _on_device, _pack_conv, _pack_lin, _pack_rgb, _pack_up2x
from .spec import TDRQVAEArch
from .swin3d import basic_layer_rows, pack_blocks

SWIN_LAYERS = ('tdswin_pre', 'tdswin_post')


class TDRQVAEEngine(Engine):
    arch_class = TDRQVAEArch

    def _repack(self):
        sd, w = self._sd, self.w
        for name, t in sd.items():
            if name.startswith(SWIN_LAYERS):
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
            elif t.dtype.is_floating_point and t.dim() == 1:
                w[name] = t.float().contiguous()
        w['codebook'] = self._f32('quantizer.codebooks.0.weight')
        self._repack_attn_qkv()
        self.swin = {p: pack_blocks(lambda k, p=p: sd.get(p + '.' + k), self.arch.stages_atten) for p in SWIN_LAYERS}

    # ------------------------------------------------------------------ blocks
    def encoder(self, x):
        """Encoder.forward (`archs/tdrqvae_arch.py:650-680`); x fp32 NCHW [F,3,H,W] -> (h [F,H/16,W/16,z], [])."""
        a = self.arch
        h = self.conv_in(x)
        for lvl in range(a.num_levels):
            C, last = a.level_ch[lvl], lvl == a.num_levels - 1
            for blk in range(a.num_res_blocks):
                # a Normalize() reads this block's output unless the stride-2 Downsample conv comes next
                more = blk < a.num_res_blocks - 1 or last
                h = self.td_resblock(h, 'encoder.down.%d.block.%d' % (lvl, blk), C,
                                     gn_next=more or a.level_has_attn[lvl])
                if a.level_has_attn[lvl]:
                    h = self.attn_block(h, 'encoder.down.%d.attn.%d' % (lvl, blk), gn_next=more)
            if not last:
                h = self._conv3(h, 'encoder.down.%d.downsample.conv' % lvl, C, stride=2, pad_lo=0, gn_out=True)
        C = a.level_ch[-1]
        h = self.td_resblock(h, 'encoder.mid.block_1', C, gn_next=True)
        h = self.attn_block(h, 'encoder.mid.attn_1', gn_next=True)
        h = self.td_resblock(h, 'encoder.mid.block_2', C, gn_next=True)
        return self._conv3(h, 'encoder.conv_out', a.z_channels, gn='encoder.norm_out'), []

    def decoder(self, z, feats=None, wgt=0.0):
        """Decoder.forward (`archs/tdrqvae_arch.py:753-784`); z [F,h,w,z_channels] bf16 -> fp32 NCHW [F,3,16h,16w]."""
        a = self.arch
        C = a.level_ch[-1]
        h = self._conv3(z, 'decoder.conv_in', C, gn_out=True)
        h = self.td_resblock(h, 'decoder.mid.block_1', C, gn_next=True)
        h = self.attn_block(h, 'decoder.mid.attn_1', gn_next=True)
        h = self.td_resblock(h, 'decoder.mid.block_2', C, gn_next=True)
        nblk = a.num_res_blocks + 1
        for lvl in reversed(range(a.num_levels)):
            C = a.level_ch[lvl]
            for blk in range(nblk):
                # a Normalize() reads this block's output unless the Upsample conv comes next
                more = blk < nblk - 1 or lvl == 0
                h = self.td_resblock(h, 'decoder.up.%d.block.%d' % (lvl, blk), C, gn_next=more or a.level_has_attn[lvl])
                if a.level_has_attn[lvl]:
                    h = self.attn_block(h, 'decoder.up.%d.attn.%d' % (lvl, blk), gn_next=more)
            if lvl != 0:
                h = self.up2x(h, 'decoder.up.%d.upsample.conv' % lvl)
        return self.decoder_out(h)

    def tdswin(self, name, z, b, t, hh, ww, out_dtype=BF):
        """tdswin_pre / tdswin_post on the latent rows z [b*t*hh*ww, E] bf16 -> new rows of out_dtype."""
        a = self.arch
        out = self._new(z.shape[0], a.embed_dim, dtype=out_dtype)
        return basic_layer_rows(z, b, t, hh, ww, self.swin[name], a.num_head, a.window_size, out=out)

    # ------------------------------------------------------------------ model methods
    def _quantise(self, x):
        """encode -> tdswin_pre -> L2 argmin of x [b,t,3,H,W].  Returns (z_e fp32 [T,E] after tdswin_pre, codes int64
        [T], z_q fp32 [T,E] codebook rows, (b, t, hh, ww))."""
        a = self.arch
        b, t, _, H, W = x.shape
        xs = x.to(self.dev, torch.float32).reshape(b * t, 3, H, W).contiguous()
        self._fusing = False
        h, _ = self.encoder(xs)
        hh, ww = H // a.down, W // a.down
        T = b * t * hh * ww
        z = self._lin(h.view(T, -1), 'quant_conv', a.embed_dim)
        z = self.tdswin('tdswin_pre', z, b, t, hh, ww, out_dtype=torch.float32)
        codes = torch.empty(T, dtype=torch.int64, device=self.dev)
        z_q = self._new(T, a.embed_dim, dtype=torch.float32)
        ops.l2_argmin_tc(z, self.w['codebook'], self._codebook_pack(), a.n_embed, codes, z_q)
        return z, codes, z_q, (b, t, hh, ww)

    @_on_device
    @torch.no_grad()
    def forward(self, x, code_only=False, force_codes=None):
        """TDRQVAE.forward (`archs/tdrqvae_arch.py:843-861`) of x [b,t,3,H,W]: (out fp32 [b,t,3,H,W], quant_loss,
        code int64 [b,t,h,w,1]); with code_only, (z_q after tdswin_post fp32 [b,t,h,w,E], quant_loss, code).
        force_codes (decoder parity checks) replaces the argmin codes before tdswin_post; loss and the returned codes
        stay those of the argmin."""
        a = self.arch
        z, codes, z_q, (b, t, hh, ww) = self._quantise(x)
        loss = (z - z_q).pow(2).mean()
        T = codes.numel()
        idx = codes if force_codes is None else force_codes.to(self.dev, torch.int64).reshape(T).contiguous()
        q16 = self._new(T, a.embed_dim)
        ops.argmax_gather(None, self.w['codebook'], None, q16, idx_in=idx)
        codes = codes.view(b, t, hh, ww, 1)
        if code_only:
            z = self.tdswin('tdswin_post', q16, b, t, hh, ww, out_dtype=torch.float32)
            return z.view(b, t, hh, ww, a.embed_dim), loss, codes
        z = self.tdswin('tdswin_post', q16, b, t, hh, ww)
        z = self._lin(z, 'post_quant_conv', a.z_channels)
        out = self.decoder(z.view(b * t, hh, ww, a.z_channels))
        return out.view(b, t, a.out_ch, hh * a.down, ww * a.down), loss, codes

    @_on_device
    @torch.no_grad()
    def codes(self, x):
        """TDRQVAE.get_codes (`:879-889`): the argmin codes of forward, [b,t,h,w,1] int64."""
        _, codes, _, (b, t, hh, ww) = self._quantise(x)
        return codes.view(b, t, hh, ww, 1)

    @_on_device
    @torch.no_grad()
    def latents(self, x):
        """(z_e = encode(x) fp32 [b*t,h,w,E], the same after tdswin_pre as forward computes it): parity checks."""
        b, t, _, H, W = x.shape
        z_e = self.encode(x.reshape(b * t, *x.shape[2:]))
        z = self._quantise(x)[0]
        return z_e, z.view(z_e.shape)
