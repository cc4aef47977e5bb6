"""Drop-in `archs/pgtformer_arch.py`: the reference's model surface over the H100 engine.

Same import path, constructor keywords and forward contract as the reference class
(`archs/pgtformer_arch.py:490-714`, built from `options/release_test_stage_IIII_*.yml ->
network_g`), so `inference.py` / `inference_cn.py` run unchanged:

    from archs.pgtformer_arch import PGTFormer
    model = PGTFormer(**network_g).cuda(); model.eval(); out = model(x, w=1)[0][1]

Parameters live in an nn.Module tree whose state_dict has exactly the reference's 961 entries
(names / shapes / dtypes, SURVEY App. D), so both checkpoint formats load with strict=True:
HF `from_pretrained` (config.json + model.safetensors) and BasicSR `.pth` `params_ema`.
forward() never runs PyTorch modules: it hands raw device pointers to libpgt_b200.so via
pgtformer_b200.engine.Engine; kernel-layout weight copies are derived caches rebuilt after
load_state_dict() / .to().  Inference only (the reference's training loop is not in its repo,
SURVEY F12); there is no CPU path.
"""
import os

import torch
import torch.nn as nn

from pgtformer_b200.registry import ARCH_REGISTRY
from pgtformer_b200.spec import build_spec
from pgtformer_b200.weights import synth_tensor

try:
    from huggingface_hub import PyTorchModelHubMixin
except Exception:                                       # pragma: no cover
    class PyTorchModelHubMixin:                         # type: ignore
        pass


class _Node(nn.Module):
    """Anonymous container: the module tree only exists to give parameters their reference names."""
    _pgt_root = None          # weak reference to the owning model (set by _materialise)

    def load_state_dict(self, state_dict, strict=True, **kw):
        # loading into a submodule (e.g. model.conditionnet.load_state_dict(...), as the reference does for the
        # face-parsing weights) must drop the root's packed-weight engine too
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        root = self._pgt_root() if self._pgt_root is not None else None
        if root is not None:
            root._invalidate()
        return r


def _materialise(root, spec, seed):
    import weakref
    rootref = weakref.ref(root)
    for name, (shape, kind, dtype) in spec.items():
        parts = name.split('.')
        node = root
        for part in parts[:-1]:
            if part not in node._modules:
                child = _Node()
                child._pgt_root = rootref
                node.add_module(part, child)
            node = node._modules[part]
        t = synth_tensor(name, shape, 'codebook' if kind == 'codebook_ema' else kind, dtype, seed)
        if kind == 'codebook_ema':
            t = t[:-1] if t.shape[0] == shape[0] + 1 else t
        if kind in ('bn_mean', 'bn_var', 'bn_count', 'rpb_index', 'zeros', 'codebook_ema'):
            node.register_buffer(parts[-1], t)
        else:
            node.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))


class _B200Model(nn.Module):
    _PGT_KEYS = ()

    def _setup(self, network_g, seed=0):
        self._network_g = network_g
        self.arch, self._spec = build_spec(network_g)
        _materialise(self, self._spec, seed)
        # embed_ema mirrors the codebook rows (tdcrqvae3_arch.py:96)
        cb = self.quantizer.codebooks._modules['0']
        cb.embed_ema.copy_(cb.weight.detach()[:-1])
        self._engine = None
        self.t = self.arch.tf
        self.code_shape = list(self.arch.code_shape)
        self.training = False

    # ---- engine cache: rebuilt whenever parameters may have changed / moved
    def _invalidate(self):
        self.__dict__['_engine'] = None

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._invalidate()
        return r

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._invalidate()
        return r

    def refresh(self):
        """Rebuilds the packed kernel-layout weights on the next forward.  load_state_dict() (on the model or any
        submodule) and .to() / .cuda() do this automatically; call it after in-place edits of parameters
        (`p.data.copy_(...)`, EMA swaps), which PyTorch gives no hook for."""
        self._invalidate()
        return self

    def engine(self):
        if self.__dict__.get('_engine') is None:
            from pgtformer_b200.engine import Engine
            dev = next(self.parameters()).device
            if dev.type != 'cuda':
                raise RuntimeError('pgtformer_b200: no CPU path — move the model to a CUDA (sm_90a) device first')
            self.__dict__['_engine'] = Engine(self._network_g, self.state_dict(), dev)
        return self.__dict__['_engine']

    def train(self, mode=True):
        """The reference's train() forgets `return self` (archs/pgtformer_arch.py:577-581), so
        `model.eval()` is used as a statement; both styles work here.  Modules stay frozen."""
        if mode:
            raise RuntimeError('pgtformer_b200 is an inference path: training mode is not supported')
        self.training = False
        return self


@ARCH_REGISTRY.register()
class TDCRQVAE3(_B200Model, PyTorchModelHubMixin):
    """Registered stage-I autoencoder (`archs/tdcrqvae3_arch.py:710-792`): forward / get_codes
    run the encoder, the nearest-codebook L2 argmin kernel and the decoder."""

    def __init__(self, *, embed_dim=64, n_embed=512, decay=0.99, loss_type='mse', latent_loss_weight=0.25,
                 bottleneck_type='rq', ddconfig=None, checkpointing=False, tf=3, **kwargs):
        super().__init__()
        assert loss_type in ['mse', 'l1']
        g = dict(kwargs)
        g.update(embed_dim=embed_dim, n_embed=n_embed, decay=decay, loss_type=loss_type,
                 latent_loss_weight=latent_loss_weight, bottleneck_type=bottleneck_type, ddconfig=ddconfig,
                 checkpointing=checkpointing, tf=tf)
        self._setup(g)

    def forward(self, input, code_only=False):
        return self.engine().forward_vq(input, code_only=code_only)

    @torch.no_grad()
    def get_codes(self, input):
        return self.engine().forward_vq(input, code_only=True)[2]


@ARCH_REGISTRY.register()
class PGTFormer(TDCRQVAE3):
    def __init__(self, ddconfig, dim_embd=512, n_head=8, n_layers=9, connect_list=['32', '64', '128', '256'],
                 fix_modules=['quantizer', 'decoder', 'conditionnet'], w=0, detach_16=True, adain=False, tf=3,
                 droprate=0.0, **kwargs):
        nn.Module.__init__(self)
        g = dict(kwargs)
        g.pop('type', None)
        g.update(ddconfig=ddconfig, dim_embd=dim_embd, n_head=n_head, n_layers=n_layers,
                 connect_list=list(connect_list), tf=tf)
        if g.get('loss_type', 'mse') not in ['mse', 'l1']:
            raise AssertionError('loss_type')
        self.fix_modules = fix_modules
        self.w = w
        self.detach_16 = detach_16
        self.adain = adain
        self.connect_list = list(connect_list)
        self.n_layers = n_layers
        self.dim_embd = dim_embd
        self.dim_mlp = dim_embd * 2
        self._setup(g)
        self.codebook_size = self.arch.n_embed
        self.quantizer_depth = self.arch.code_shape[-1]
        # replay the forward from a CUDA graph (static output tensors!) — opt-in: attribute or PGT_CUDA_GRAPH=1
        self.cuda_graph = os.environ.get('PGT_CUDA_GRAPH', '0') == '1'

    def forward(self, x, w=None, detach_16=True, code_only=None, adain=None, force_codes=None):
        """`archs/pgtformer_arch.py:598-714`: returns (out, logits, lq_feat_nhwc), or
        (logits, lq_feat_nhwc) when code_only.  `detach_16` only matters for autograd and is
        accepted for signature compatibility.  `force_codes` (extension) teacher-forces the code
        indices for decoder parity checks."""
        if w is None:
            w = self.w
        if adain is None:
            adain = self.adain
        if self.cuda_graph and not code_only and force_codes is None:
            return self.engine().forward_graphed(x, w=w, adain=bool(adain))
        return self.engine().forward(x, w=w, adain=bool(adain), code_only=bool(code_only), force_codes=force_codes)

    def forward_vq(self, input, code_only=False):
        """The inherited TDCRQVAE3.forward on this model's weights (the L2-argmin path)."""
        return self.engine().forward_vq(input, code_only=code_only)
