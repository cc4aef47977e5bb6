"""Drop-in `archs/codeformer_arch.py`: the reference's CodeFormer (`archs/codeformer_arch.py:229-366`) over the H100 engine
(pgtformer_b200/vqgan.py), registered as 'CodeFormer' (the reference leaves it unregistered, as it does PGTFormer).

Same constructor keywords, forward defaults and returns, and the reference's state-dict names, shapes and dtypes
(loads with strict=True):

    from archs.codeformer_arch import CodeFormer
    model = CodeFormer().cuda().eval(); model.load_state_dict(ckpt['params_ema'])
    out, logits, lq_feat = model(x, w=0.5, adain=True)           # x [b, 3, 512, 512] in [-1, 1]

Inference only, no CPU path; 512^2 inputs only, as in the reference (position_emb has one row per token of the 16 x 16
latent, and forward reshapes the codes to [b, 16, 16, 256]).  fix_modules and detach_16 only matter for training and
have no effect here.  Codes are the first maximum of the fp32 logits; the reference's topk(softmax(logits), 1) can pick a
later index where two logits are close enough that their probabilities round to the same fp32 value."""
import torch

from archs.vqgan_arch import VQAutoEncoder
from pgtformer_b200.registry import ARCH_REGISTRY


@ARCH_REGISTRY.register()
class CodeFormer(VQAutoEncoder):
    _codeformer = True

    def __init__(self, dim_embd=512, n_head=8, n_layers=9, codebook_size=1024, latent_size=256,
                 connect_list=['32', '64', '128', '256'], fix_modules=['quantize', 'generator'], img_size=512, nf=64,
                 ch_mult=[1, 2, 2, 4, 4, 8], quantizer="nearest", res_blocks=2, attn_resolutions=[16], emb_dim=256,
                 w=0, detach_16=True, adain=False, last_silu=False):
        super().__init__(img_size, nf, ch_mult, quantizer, res_blocks, attn_resolutions, codebook_size, emb_dim=emb_dim,
                         last_silu=last_silu, _transformer=dict(dim_embd=dim_embd, n_head=n_head, n_layers=n_layers,
                                                                latent_size=latent_size,
                                                                connect_list=list(connect_list)))
        self.fix_modules = fix_modules
        self.w = w
        self.detach_16 = detach_16
        self.adain = adain
        self.connect_list = connect_list
        self.n_layers = n_layers
        self.dim_embd = dim_embd
        self.dim_mlp = dim_embd * 2

    def _engine_class(self):
        from pgtformer_b200.vqgan import CodeFormerEngine
        return CodeFormerEngine

    def forward(self, x, w=None, detach_16=True, code_only=None, adain=None, force_codes=None):
        """(out fp32 [b,3,512,512], logits fp32 [b, 256, codebook_size], lq_feat fp32 [b, 256, 16, 16]), or
        (logits, lq_feat) with code_only.  `force_codes` (extension, int64 [b, 256]) teacher-forces the codes for
        decoder parity checks."""
        if w is None:
            w = self.w
        if adain is None:
            adain = self.adain
        x = self._images(x)
        if x.shape[2] != self.resolution or x.shape[3] != self.resolution:
            raise ValueError('CodeFormer takes [b, 3, %d, %d] images, got %s'
                             % (self.resolution, self.resolution, tuple(x.shape)))
        if force_codes is not None:
            b = x.shape[0]
            if not torch.is_tensor(force_codes) or force_codes.numel() != b * self.arch.latent_size or \
                    force_codes.dtype.is_floating_point:
                raise ValueError('force_codes must be integer codes [b, %d]' % self.arch.latent_size)
            lo, hi = torch.aminmax(force_codes)
            if int(lo) < 0 or int(hi) >= self.codebook_size:
                raise IndexError('code out of range [0, %d)' % self.codebook_size)
            return self.engine().forward(x, w=float(w), adain=bool(adain), code_only=bool(code_only),
                                         force_codes=force_codes)
        return self._run('forward', x, w=float(w), adain=bool(adain), code_only=bool(code_only))
