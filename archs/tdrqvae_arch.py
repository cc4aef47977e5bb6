"""Drop-in `archs/tdrqvae_arch.py`: the reference's registered TDRQVAE (`archs/tdrqvae_arch.py:787-976`) over the H100
engine (pgtformer_b200/tdrqvae.py).

Same import path, constructor keywords and method contracts as the reference class, and the reference's state-dict
names, shapes and dtypes (the `relative_position_index` buffers of tdswin_pre / tdswin_post included), so a reference
checkpoint loads with strict=True:

    from archs.tdrqvae_arch import TDRQVAE
    model = TDRQVAE(**network_g).cuda().eval(); out, quant_loss, code = model(x)     # x [b, t, 3, H, W]

Inference only, no CPU path.  Configurations the kernels cannot run raise ValueError at construction (spec.TDRQVAEArch).
Not provided: the training methods (compute_loss, get_recon_imgs, get_last_layer) and forward_partial_code, which fails
in the reference (get_codes returns 5-D codes, embed_partial_code asserts 4-D ones, `:532,974-975`)."""
import math

import torch
import torch.nn as nn

from archs.pgtformer_arch import PyTorchModelHubMixin, _B200Model, _materialise, _shape
from pgtformer_b200.registry import ARCH_REGISTRY
from pgtformer_b200.spec import build_tdrqvae_spec


@ARCH_REGISTRY.register()
class TDRQVAE(_B200Model, PyTorchModelHubMixin):
    def __init__(self, *, embed_dim=64, n_embed=512, decay=0.99, loss_type='mse', latent_loss_weight=0.25,
                 bottleneck_type='rq', ddconfig=None, checkpointing=False, tf=7, **kwargs):
        nn.Module.__init__(self)
        assert loss_type in ['mse', 'l1']
        if bottleneck_type != 'rq':
            raise ValueError("invalid 'bottleneck_type' (must be 'rq')")
        g = dict(kwargs)
        for k in ('latent_shape', 'code_shape', 'shared_codebook', 'restart_unused_codes'):
            g[k] = kwargs[k]                                  # KeyError when missing, as in the reference (:816-819)
        g.pop('type', None)
        g.update(embed_dim=embed_dim, n_embed=n_embed, decay=decay, loss_type=loss_type,
                 latent_loss_weight=latent_loss_weight, bottleneck_type=bottleneck_type, ddconfig=ddconfig,
                 checkpointing=checkpointing, tf=tf)
        self._network_g = g
        self.arch, self._spec = build_tdrqvae_spec(g)
        _materialise(self, self._spec, 0)
        self._engine = None
        self.t = tf                                           # forward never reads it: b, t come from the input
        self.code_shape = kwargs['code_shape']
        self.loss_type = loss_type
        self.latent_loss_weight = latent_loss_weight
        self.training = False

    def _engine_class(self):
        from pgtformer_b200.tdrqvae import TDRQVAEEngine
        return TDRQVAEEngine

    # ---- host-side argument checks (before any launch)
    def _clips(self, x):
        """[b, t, 3, H, W], any b, t >= 1, H and W multiples of 64."""
        if not torch.is_tensor(x) or x.dim() != 5:
            raise ValueError('expected clips [b, t, 3, H, W], got %s' % (_shape(x),))
        b, t, C, H, W = x.shape
        if b == 0 or t == 0 or C != 3 or H == 0 or W == 0 or H % 64 or W % 64:
            raise ValueError('expected clips [b, t, 3, H, W] with H, W multiples of 64, got %s' % (tuple(x.shape),))
        return x

    def _frames(self, x):
        """[F, 3, H, W], F >= 1, H and W multiples of 64 (encode and get_soft_codes take frames, as in the reference)."""
        if not torch.is_tensor(x) or x.dim() != 4:
            raise ValueError('expected frames [F, 3, H, W], got %s' % (_shape(x),))
        Fr, C, H, W = x.shape
        if Fr == 0 or C != 3 or H == 0 or W == 0 or H % 64 or W % 64:
            raise ValueError('expected frames [F, 3, H, W] with H, W multiples of 64, got %s' % (tuple(x.shape),))
        return x

    def _check_latent(self, Fr, h, w):
        if Fr == 0 or h == 0 or w == 0 or h % 4 or w % 4:
            raise ValueError('expected a latent map of multiples of 4 (frames multiples of 64), got [%d, %d, %d]'
                             % (Fr, h, w))

    # ---- the reference's methods (`archs/tdrqvae_arch.py:843-976`)
    def forward(self, input, code_only=False):
        """(out [b,t,3,H,W], quant_loss, code [b,t,h,w,1]); with code_only, (z_q after tdswin_post [b,t,h,w,E],
        quant_loss, code)."""
        x = self._clips(input)
        return self._run('forward', x, code_only=bool(code_only))

    @torch.no_grad()
    def get_codes(self, input):
        """Codes [b,t,h,w,1] of the tdswin_pre output (the codes forward returns)."""
        x = self._clips(input)
        return self._run('codes', x)

    @torch.no_grad()
    def get_codesbt(self, input):
        """get_codes as [b*t,h,w,1]."""
        code = self.get_codes(input)
        return code.view(-1, *code.shape[2:])

    @torch.no_grad()
    def encode(self, x):
        """z_e = quant_conv(Encoder(x)) of frames [F,3,H,W] as NHWC fp32 [F, H/16, W/16, embed_dim]; no Swin layer."""
        x = self._frames(x)
        return self._run('encode', x)

    @torch.no_grad()
    def decode(self, z_q):
        """post_quant_conv + Decoder of NHWC z_q [F, h, w, embed_dim] -> fp32 [F, 3, 16h, 16w]; no Swin layer."""
        if not torch.is_tensor(z_q) or z_q.dim() != 4 or z_q.shape[-1] != self.arch.embed_dim or \
                not z_q.dtype.is_floating_point:
            raise ValueError('expected z_q [F, h, w, %d] floating point, got %s' % (self.arch.embed_dim, _shape(z_q)))
        self._check_latent(*z_q.shape[:3])
        return self._run('decode', z_q)

    @torch.no_grad()
    def decode_code(self, code):
        """Codebook rows of the int codes [F, h, w, 1], decoded to frames without tdswin_post."""
        self._check_code(code)
        self._check_latent(*code.shape[:3])
        return self._run('decode_code', code)

    @torch.no_grad()
    def get_soft_codes(self, xs, temp=1.0, stochastic=False):
        """(soft_code [F, h, w, 1, n_embed] fp32 = softmax(-||z_e - e_k||^2 / temp), code [F, h, w, 1] int64) on
        z_e = encode(xs), without tdswin_pre (as in the reference, `:904-910`)."""
        try:
            t = float(temp)
        except (TypeError, ValueError):
            raise ValueError('temp must be a finite number > 0, got %r' % (temp,)) from None
        if not math.isfinite(t) or t <= 0.0:
            raise ValueError('temp must be a finite number > 0, got %r' % (temp,))
        x = self._frames(xs)
        eng = self.engine()
        z_e = eng.encode(x)
        Fr, h, w, E = z_e.shape
        p, code = eng.soft_codes(z_e.view(-1, E), t, stochastic=bool(stochastic))
        return p.view(Fr, h, w, 1, -1), code.view(Fr, h, w, 1)
