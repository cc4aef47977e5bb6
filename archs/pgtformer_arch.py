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
import math
import os

import torch
import torch.nn as nn

from pgtformer_b200.registry import ARCH_REGISTRY
from pgtformer_b200.spec import build_spec
from pgtformer_b200.weights import synth_state_dict

try:
    from huggingface_hub import PyTorchModelHubMixin
except Exception:                                       # pragma: no cover
    class PyTorchModelHubMixin:                         # type: ignore
        pass


def _shape(x):
    return tuple(x.shape) if torch.is_tensor(x) else type(x).__name__


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
    """root's module tree of spec's entries, holding synth_state_dict's tensors (each embed_ema its codebook's rows)."""
    import weakref
    rootref = weakref.ref(root)
    sd = synth_state_dict(spec, seed)
    for name, (shape, kind, dtype) in spec.items():
        if spec.alias_of(name):
            continue
        parts = name.split('.')
        node = root
        for part in parts[:-1]:
            if part not in node._modules:
                child = _Node()
                child._pgt_root = rootref
                node.add_module(part, child)
            node = node._modules[part]
        t = sd[name]
        if kind in ('bn_mean', 'bn_var', 'bn_count', 'rpb_index', 'zeros', 'codebook_ema'):
            node.register_buffer(parts[-1], t)
        else:
            node.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))
    # a shared codebook is the same module under every depth, as in the reference's ModuleList: state_dict() repeats its
    # keys and load_state_dict(strict=True) loads each copy into the one tensor in turn (the last one wins)
    for alias, target in spec.module_aliases.items():
        *path, leaf = alias.split('.')
        parent, node = root, root
        for part in path:
            parent = parent._modules[part]
        for part in target.split('.'):
            node = node._modules[part]
        parent.add_module(leaf, node)


class _B200Model(nn.Module):
    _PGT_KEYS = ()
    # replay the model's calls from CUDA graphs (Engine.graphed): their outputs are then the graphs' static tensors, to
    # be consumed before the next call.  Off by default; PGTFormer reads PGT_CUDA_GRAPH and replays its forward only.
    cuda_graph = False
    _graph_calls = True       # whether cuda_graph covers the codec calls routed through _run (not for PGTFormer)

    def _setup(self, network_g, seed=0):
        self._network_g = network_g
        self.arch, self._spec = build_spec(network_g)
        _materialise(self, self._spec, seed)
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
            dev = next(self.parameters()).device
            if dev.type != 'cuda':
                raise RuntimeError('pgtformer_b200: no CPU path — move the model to a CUDA (sm_90a) device first')
            self.__dict__['_engine'] = self._engine_class()(self._network_g, self.state_dict(), dev)
        return self.__dict__['_engine']

    def _engine_class(self):
        from pgtformer_b200.engine import Engine
        return Engine

    def _run(self, name, *tensors, writes=(), **scalars):
        """The engine's method `name` on the tensors and scalars: eager, or with cuda_graph replayed from the engine's
        graph for this key (Engine.graphed; `writes`: the tensors the method updates in place).  The caller has checked
        the arguments on the host."""
        eng = self.engine()
        if self.cuda_graph and self._graph_calls:
            return eng.graphed(getattr(eng, name), tensors, writes=writes, **scalars)
        return getattr(eng, name)(*tensors, **scalars)

    # ---- code helpers shared by the codecs.  Arguments are checked on the host before any launch: bad shapes
    # raise ValueError, depth d's codes outside [0, n_embeds[d]] IndexError (index n_embeds[d] is the codebook's
    # padding row, which nn.Embedding accepts).
    def _check_code(self, code):
        if not torch.is_tensor(code) or code.dim() != 4 or code.shape[-1] != self.code_shape[-1] or \
                code.dtype.is_floating_point or code.dtype.is_complex or code.dtype == torch.bool:
            raise ValueError('expected integer codes [F, h, w, %d], got %s %s'
                             % (self.code_shape[-1], _shape(code), getattr(code, 'dtype', '')))
        if code.numel() > 0:
            lo, hi = torch.stack(torch.aminmax(code.reshape(-1, code.shape[-1]), dim=0)).tolist()    # one host sync
            for d, n in enumerate(self.arch.n_embeds):
                if lo[d] < 0 or hi[d] > n:
                    raise IndexError('depth %d: code out of range [0, %d]: min %d, max %d' % (d, n, lo[d], hi[d]))

    @torch.no_grad()
    def get_code_emb_with_depth(self, code):
        """(codebook rows [F, h, w, D, embed_dim] fp32, None), as RQBottleneck.embed_code_with_depth returns them."""
        self._check_code(code)
        Fr, h, w, d = code.shape
        return self.engine().embed_code_with_depth(code).view(Fr, h, w, d, self.arch.embed_dim), None

    @torch.no_grad()
    def decode_partial_code(self, code, code_idx, decode_type='select'):
        """RQBottleneck.embed_partial_code + decode (`archs/tdcrqvae3_arch.py:394-426, 855-863`): 'select' decodes the
        code rows of depth code_idx alone, 'add' the sum of depths 0 .. code_idx; with one codebook both are
        decode_code."""
        self._check_code(code)
        assert code_idx < code.shape[-1]
        if decode_type not in ('select', 'add'):
            raise NotImplementedError(f"{decode_type} is not implemented in partial decoding")
        if code.shape[-1] == 1:
            self._check_latent(*code.shape[:3])
            return self.engine().decode_code(code)
        if isinstance(code_idx, bool) or not isinstance(code_idx, int) or code_idx < 0:
            raise ValueError('code_idx must be an int in [0, %d), got %r' % (code.shape[-1], code_idx))
        self._check_latent(*code.shape[:3])
        eng = self.engine()
        Fr, h, w, _ = code.shape
        z_q = eng.embed_code(code, code_idx if decode_type == 'select' else 0, code_idx)
        return eng.decode(z_q.view(Fr, h, w, self.arch.embed_dim))

    def train(self, mode=True):
        """The reference's train() forgets `return self` (archs/pgtformer_arch.py:577-581), so
        `model.eval()` is used as a statement; both styles work here.  Modules stay frozen."""
        if mode:
            raise RuntimeError('pgtformer_b200 is an inference path: training mode is not supported')
        self.training = False
        return self


@ARCH_REGISTRY.register()
class TDCRQVAE3(_B200Model, PyTorchModelHubMixin):
    """Registered stage-I autoencoder (`archs/tdcrqvae3_arch.py:710-872`): forward / get_codes run the encoder, the
    residual quantiser (one exact nearest-codebook L2 argmin per code depth, `code_shape[2]`; separate codebooks, or one
    shared by every depth with `shared_codebook=True`) and the decoder; encode / decode / decode_code / get_soft_codes and the partial-
    code methods expose the codec's parts (PGTFormer inherits them, as in the reference)."""

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
        x = self._frames(input)
        return self._run('forward_vq', x, code_only=bool(code_only))

    @torch.no_grad()
    def get_codes(self, input):
        x = self._frames(input)
        return self._run('forward_vq', x, code_only=True)[2]

    # ---- the rest of the stage-I codec surface (`archs/tdcrqvae3_arch.py:774-872`) at any quantiser depth; arguments are
    # checked on the host before any launch (see _B200Model._check_code).
    def _frames(self, x):
        """[b, t, 3, H, W] (the reference's form) or [b*t, 3, H, W] -> [b*t, 3, H, W]."""
        if not torch.is_tensor(x) or x.dim() not in (4, 5):
            raise ValueError('expected frames [b, t, 3, H, W] or [b*t, 3, H, W], got %s' % (_shape(x),))
        if x.dim() == 5:
            x = x.reshape(-1, *x.shape[2:])
        Fr, C, H, W = x.shape
        if C != 3 or Fr == 0 or Fr % self.t != 0 or H % 64 != 0 or W % 64 != 0 or H == 0 or W == 0:
            raise ValueError('expected %d-frame clips of 3 x H x W with H, W multiples of 64, got %s'
                             % (self.t, tuple(x.shape)))
        return x

    def _check_latent(self, Fr, h, w):
        if Fr == 0 or Fr % self.t != 0 or h == 0 or w == 0 or h % 4 != 0 or w % 4 != 0:
            raise ValueError('expected %d-frame clips with a latent map of multiples of 4 (frames multiples of 64), '
                             'got [%d, %d, %d]' % (self.t, Fr, h, w))

    @torch.no_grad()
    def encode(self, x):
        """z_e = quant_conv(Encoder(x)) as NHWC fp32 [b*t, H/16, W/16, embed_dim]."""
        x = self._frames(x)
        return self._run('encode', x)

    @torch.no_grad()
    def decode(self, z_q):
        """post_quant_conv + Decoder.forward (no SFT fusion) of NHWC z_q [F, h, w, embed_dim] -> fp32 [F, 3, 16h, 16w]."""
        if not torch.is_tensor(z_q) or z_q.dim() != 4 or z_q.shape[-1] != self.arch.embed_dim or \
                not z_q.dtype.is_floating_point:
            raise ValueError('expected z_q [F, h, w, %d] floating point, got %s' % (self.arch.embed_dim, _shape(z_q)))
        self._check_latent(*z_q.shape[:3])
        return self._run('decode', z_q)

    @torch.no_grad()
    def decode_code(self, code):
        """The depth sum of the code rows of the int codes [F, h, w, D] (any h, w the decoder takes), decoded to frames."""
        self._check_code(code)
        self._check_latent(*code.shape[:3])
        return self._run('decode_code', code)

    @torch.no_grad()
    def forward_partial_code(self, xs, code_idx, decode_type='select'):
        x = self._frames(xs)
        code = self.engine().forward_vq(x, code_only=True)[2]
        return self.decode_partial_code(code, code_idx, decode_type)

    @torch.no_grad()
    def get_soft_codes(self, xs, temp=1.0, stochastic=False):
        """(soft_code [F, h, w, D, n_embed] fp32 = softmax(-||r_d - e_k||^2 / temp) over depth d's codebook, code
        [F, h, w, D] int64), r_d the residual the earlier depths' codes left: the exact nearest code (== get_codes), or
        with stochastic=True one draw per token and depth from its soft_code row."""
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
        D = self.code_shape[-1]
        return p.view(Fr, h, w, D, -1), code.view(Fr, h, w, D)


@ARCH_REGISTRY.register()
class PGTFormer(TDCRQVAE3):
    _graph_calls = False      # cuda_graph replays forward alone: the inherited codec methods keep fresh outputs

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
        (logits, lq_feat_nhwc) when code_only; logits are [b*3, h, w, D, codebook_size].  `detach_16` only
        matters for autograd and is accepted for signature compatibility.  `force_codes` (extension, int64
        [b*3, h, w, D]) teacher-forces the code indices for decoder parity checks."""
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
