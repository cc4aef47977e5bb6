"""Drop-in `archs/vqgan_arch.py`: the reference's registered VQAutoEncoder (`archs/vqgan_arch.py:344-414`) over the H100
engine (pgtformer_b200/vqgan.py).

Same import path, constructor keywords and forward contract as the reference class, and the reference's state-dict names,
shapes and dtypes, so a reference checkpoint loads with strict=True:

    from archs.vqgan_arch import VQAutoEncoder
    model = VQAutoEncoder(model_path='vqgan.pth').cuda().eval(); out, codebook_loss, quant_stats = model(x)

Inference only, no CPU path.  Configurations the kernels cannot run raise ValueError at construction (spec.VQGANArch):
the Gumbel quantiser, nf != 64, level widths that are not multiples of 32, AttnBlock widths the attention kernel does not
take.  Not provided: get_last_layer (training) and VQGANDiscriminator."""
import weakref

import torch
import torch.nn as nn

from archs.pgtformer_arch import _B200Model, _Node, _materialise, _shape
from pgtformer_b200.registry import ARCH_REGISTRY
from pgtformer_b200.spec import build_vqgan_spec


def _load_model_path(model, model_path):
    """`params_ema`, else `params`, else ValueError, as the reference loads model_path (`archs/vqgan_arch.py:393-402`)."""
    chkpt = torch.load(model_path, map_location='cpu')
    if 'params_ema' in chkpt:
        model.load_state_dict(chkpt['params_ema'])
    elif 'params' in chkpt:
        model.load_state_dict(chkpt['params'])
    else:
        raise ValueError('Wrong params!')


class _VectorQuantizer(_Node):
    """`quantize`: holds `embedding.weight` and the `usage` buffer, with VectorQuantizer's usage methods
    (`archs/vqgan_arch.py:35-40`); the quantiser itself runs in the engine."""

    def __init__(self, codebook_size):
        super().__init__()
        self.codebook_size = codebook_size
        # a non-persistent int32 buffer every eval forward adds its code counts to (`:33, 61-63`)
        self.register_buffer('usage', torch.zeros(codebook_size, dtype=torch.int), persistent=False)

    def reset_usage(self):
        self.usage = self.usage * 0

    def get_usage(self):
        return 1.0 * (self.codebook_size - (self.usage == 0).sum()) / self.codebook_size


@ARCH_REGISTRY.register()
class VQAutoEncoder(_B200Model):
    _codeformer = False

    def __init__(self, img_size=512, nf=64, ch_mult=[1, 2, 2, 4, 4, 8], quantizer="nearest", res_blocks=2,
                 attn_resolutions=[16], codebook_size=1024, emb_dim=256, beta=0.25, gumbel_straight_through=False,
                 gumbel_kl_weight=1e-8, model_path=None, last_silu=False, _transformer=None):
        nn.Module.__init__(self)
        g = dict(img_size=img_size, nf=nf, ch_mult=list(ch_mult), quantizer=quantizer, res_blocks=res_blocks,
                 attn_resolutions=list(attn_resolutions), codebook_size=codebook_size, emb_dim=emb_dim, beta=beta,
                 last_silu=last_silu, **(_transformer or {}))
        self._network_g = g
        self.arch, self._spec = build_vqgan_spec(g, self._codeformer)
        _materialise(self, self._spec, 0)
        q = _VectorQuantizer(codebook_size)                   # takes the place (and the order) of the plain node
        q._pgt_root = weakref.ref(self)
        q.add_module('embedding', self.quantize.embedding)
        self._modules['quantize'] = q
        self._engine = None
        self.in_channels = 3
        self.nf = nf
        self.n_blocks = res_blocks
        self.codebook_size = codebook_size
        self.embed_dim = emb_dim
        self.ch_mult = ch_mult
        self.resolution = img_size
        self.attn_resolutions = attn_resolutions
        self.quantizer_type = quantizer
        self.beta = beta
        self.training = False
        if model_path is not None:
            _load_model_path(self, model_path)

    def _engine_class(self):
        from pgtformer_b200.vqgan import VQGANEngine
        return VQGANEngine

    def _images(self, x):
        """[b, 3, H, W], b >= 1, H and W multiples of 4 * 2^(levels - 1) (a latent of multiples of 4), checked on the
        host before any launch."""
        m = 4 * self.arch.down
        if not torch.is_tensor(x) or x.dim() != 4 or not x.dtype.is_floating_point:
            raise ValueError('expected images [b, 3, H, W], got %s' % (_shape(x),))
        b, c, H, W = x.shape
        if b == 0 or c != 3 or H == 0 or W == 0 or H % m or W % m:
            raise ValueError('expected images [b, 3, H, W] with H, W multiples of %d, got %s' % (m, tuple(x.shape)))
        return x

    def forward(self, x, code_only=False):
        """(out fp32 [b,3,H,W], codebook_loss, quant_stats), or (quant fp32 [b, emb_dim, h, w], codebook_loss,
        quant_stats) with code_only; quant_stats as VectorQuantizer.forward returns it (`archs/vqgan_arch.py:78-84`)."""
        x = self._images(x)
        eng = self.engine()
        usage = self.quantize.usage
        if usage.device != eng.dev:
            raise RuntimeError('quantize.usage is on %s, the model on %s' % (usage.device, eng.dev))
        # a replay adds its counts to the buffer held now (reset_usage() replaces it), through the graph's own copy
        return self._run('counted_forward', x, usage, writes=(1,), code_only=bool(code_only))
