"""Drop-in `archs/rqvae_arch.py`: the reference's registered RQVAE (`archs/rqvae_arch.py:779-931`) over the H100 engine
(pgtformer_b200/rqvae.py).

Same import path, constructor keywords and method contracts as the reference class, and the reference's state-dict
names, shapes and dtypes, so a reference checkpoint loads with strict=True:

    from archs.rqvae_arch import RQVAE
    model = RQVAE(**network_g).cuda().eval(); out, quant_loss, code = model(x)        # x [B, 3, H, W], code [B, h, w, D]

Inference only, no CPU path.  Configurations the kernels cannot run, and those the reference accepts but fails on at
forward, raise ValueError at construction (spec.RQVAEArch).  Not provided: the training methods (compute_loss,
get_recon_imgs, get_last_layer) and the codebooks' EMA updates."""
import math

import torch
import torch.nn as nn

from archs.pgtformer_arch import PyTorchModelHubMixin, _B200Model, _materialise, _shape
from pgtformer_b200.registry import ARCH_REGISTRY
from pgtformer_b200.spec import build_rqvae_spec


@ARCH_REGISTRY.register()
class RQVAE(_B200Model, PyTorchModelHubMixin):
    def __init__(self, *, embed_dim=64, n_embed=512, decay=0.99, loss_type='mse', latent_loss_weight=0.25,
                 bottleneck_type='rq', ddconfig=None, checkpointing=False, **kwargs):
        nn.Module.__init__(self)
        assert loss_type in ['mse', 'l1']
        if bottleneck_type != 'rq':
            raise ValueError("invalid 'bottleneck_type' (must be 'rq')")
        g = dict(kwargs)
        for k in ('latent_shape', 'code_shape', 'shared_codebook', 'restart_unused_codes'):
            g[k] = kwargs[k]                                  # KeyError when missing, as in the reference (:807-810)
        g.pop('type', None)
        g.update(embed_dim=embed_dim, n_embed=n_embed, decay=decay, loss_type=loss_type,
                 latent_loss_weight=latent_loss_weight, bottleneck_type=bottleneck_type, ddconfig=ddconfig,
                 checkpointing=checkpointing)
        self._network_g = g
        self.arch, self._spec = build_rqvae_spec(g)
        _materialise(self, self._spec, 0)
        self._engine = None
        self.code_shape = kwargs['code_shape']
        self.loss_type = loss_type
        self.latent_loss_weight = latent_loss_weight
        self.training = False

    def _engine_class(self):
        from pgtformer_b200.rqvae import RQVAEEngine
        return RQVAEEngine

    # ---- host-side argument checks (before any launch)
    def _images(self, x, dims=4):
        """[B, 3, H, W] (or [b, t, 3, H, W] with dims=5), B >= 1, H and W multiples of max(64, 4 * 2^(levels - 1)): a
        latent of multiples of 4, and frames of multiples of 64 as for TDRQVAE, whose encoder / decoder these are."""
        m = max(64, 4 * self.arch.down)
        if not torch.is_tensor(x) or x.dim() != dims or not x.dtype.is_floating_point:
            raise ValueError('expected images [%s3, H, W], got %s' % ('b, t, ' if dims == 5 else 'B, ', _shape(x)))
        C, H, W = x.shape[-3:]
        if x.numel() == 0 or C != 3 or H % m or W % m:
            raise ValueError('expected images with 3 channels and H, W multiples of %d, got %s' % (m, tuple(x.shape)))
        return x

    def _check_latent(self, B, h, w):
        if B == 0 or h == 0 or w == 0 or h % 4 or w % 4:
            raise ValueError('expected a latent map of multiples of 4, got [%d, %d, %d]' % (B, h, w))

    # ---- the reference's methods (`archs/rqvae_arch.py:828-931`)
    def forward(self, xs, code_only=False):
        """(out fp32 [B,3,H,W], quant_loss, code int64 [B,h,w,D]); with code_only, (z_q fp32 [B,h,w,embed_dim],
        quant_loss, code)."""
        x = self._images(xs)
        return self._run('forward_vq', x, code_only=bool(code_only))

    @torch.no_grad()
    def encode(self, x):
        """z_e = quant_conv(Encoder(x)) as NHWC fp32 [B, h, w, embed_dim]."""
        x = self._images(x)
        return self._run('encode', x)

    @torch.no_grad()
    def decode(self, z_q):
        """post_quant_conv + Decoder of NHWC z_q [B, h, w, embed_dim] -> fp32 [B, 3, f h, f w]."""
        if not torch.is_tensor(z_q) or z_q.dim() != 4 or z_q.shape[-1] != self.arch.embed_dim or \
                not z_q.dtype.is_floating_point:
            raise ValueError('expected z_q [B, h, w, %d] floating point, got %s' % (self.arch.embed_dim, _shape(z_q)))
        self._check_latent(*z_q.shape[:3])
        return self._run('decode', z_q)

    @torch.no_grad()
    def get_codes(self, xs):
        """Codes [B, h, w, D] int64 (those forward returns)."""
        x = self._images(xs)
        return self._run('forward_vq', x, code_only=True)[2]

    @torch.no_grad()
    def get_codesbt(self, xs):
        """get_codes of clips [b, t, 3, H, W] as [b*t, h, w, D]."""
        x = self._images(xs, dims=5)
        return self._run('forward_vq', x.reshape(-1, *x.shape[2:]), code_only=True)[2]

    @torch.no_grad()
    def get_soft_codes(self, xs, temp=1.0, stochastic=False):
        """(soft_code [B, h, w, D, n_embed] fp32 = softmax(-||r_d - e_k||^2 / temp) over depth d's codebook, code
        [B, h, w, D] int64), r_d the residual the earlier depths' codes left: the exact nearest code (== get_codes), or
        with stochastic=True one draw per token and depth from its soft_code row.  The reference concatenates the
        depths' soft codes, so codebooks of different sizes raise ValueError (the reference fails in torch.cat)."""
        try:
            t = float(temp)
        except (TypeError, ValueError):
            raise ValueError('temp must be a finite number > 0, got %r' % (temp,)) from None
        if not math.isfinite(t) or t <= 0.0:
            raise ValueError('temp must be a finite number > 0, got %r' % (temp,))
        if len(set(self.arch.n_embeds)) != 1:
            raise ValueError('get_soft_codes needs codebooks of one size, got n_embed %s' % (list(self.arch.n_embeds),))
        x = self._images(xs)
        eng = self.engine()
        z_e = eng.encode(x)
        B, h, w, E = z_e.shape
        p, code = eng.soft_codes(z_e.view(-1, E), t, stochastic=bool(stochastic))
        D = self.arch.depth
        return p.view(B, h, w, D, -1), code.view(B, h, w, D)

    @torch.no_grad()
    def decode_code(self, code):
        """The depth sum of the code rows of the int codes [B, h, w, D], decoded to images."""
        self._check_code(code)
        self._check_latent(*code.shape[:3])
        return self._run('decode_code', code)

    @torch.no_grad()
    def forward_partial_code(self, xs, code_idx, decode_type='select'):
        """decode_partial_code of get_codes(xs), both eager."""
        x = self._images(xs)
        code = self.engine().forward_vq(x, code_only=True)[2]
        return self.decode_partial_code(code, code_idx, decode_type)
