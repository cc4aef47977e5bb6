"""Deterministic synthetic checkpoints (the kernel-layout repack is Engine._repack, pgtformer_b200/engine.py).

No trained weights are reachable offline (SURVEY F10), so every test / bench uses a synthetic
state dict that is a pure function of (name, shape, kind, seed): independent of module
construction order, hence reproducible wherever the tests run (without the reference) and
loadable into the reference with `load_state_dict(strict=True)` to mint golden vectors.
Scales follow PyTorch's default init (U(+-1/sqrt(fan_in))) so activations stay O(1); biases,
norm affine terms and the relative-position tables are deliberately non-trivial so that index /
bias mistakes are visible in parity tests.
"""
import hashlib
import math

import torch

from .spec import WINDOW


def relative_position_index(window=WINDOW):
    """[N,N] int64 index (N = D*Wh*Ww) into the (2D-1)(2Wh-1)(2Ww-1)-row bias table: offset
    (dd+D-1)*(2Wh-1)*(2Ww-1) + (dh+Wh-1)*(2Ww-1) + (dw+Ww-1) for tokens ordered (d, h, w).  The default (3,4,4) window
    gives PGTFormer's [48,48] index (`modules/rstt_layers.py:163-184`), (5,5,5) TDRQVAE's Video-Swin [125,125] one
    (`modules/swin.py:117-130`)."""
    D, Wh, Ww = window
    d = torch.arange(D).view(D, 1, 1).expand(D, Wh, Ww).reshape(-1)
    h = torch.arange(Wh).view(1, Wh, 1).expand(D, Wh, Ww).reshape(-1)
    w = torch.arange(Ww).view(1, 1, Ww).expand(D, Wh, Ww).reshape(-1)
    rd = d[:, None] - d[None, :] + (D - 1)
    rh = h[:, None] - h[None, :] + (Wh - 1)
    rw = w[:, None] - w[None, :] + (Ww - 1)
    return (rd * (2 * Wh - 1) * (2 * Ww - 1) + rh * (2 * Ww - 1) + rw).to(torch.int64)


def _gen(name, seed):
    h = hashlib.sha256(('%d:%s' % (seed, name)).encode()).digest()
    g = torch.Generator(device='cpu')
    g.manual_seed(int.from_bytes(h[:8], 'little') & 0x7FFFFFFFFFFFFFFF)
    return g


def synth_tensor(name, shape, kind, dtype, seed=0, window=None):
    """window: the (D, H, W) attention window of an 'rpb_index' buffer (Spec.windows; default spec.WINDOW)."""
    g = _gen(name, seed)
    if kind in ('conv_w', 'linear_w'):
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        bound = 1.0 / math.sqrt(fan_in)
        return (torch.rand(shape, generator=g) * 2 - 1) * bound
    if kind == 'bias':
        return (torch.rand(shape, generator=g) * 2 - 1) * 0.05
    if kind == 'norm_w':
        return 1.0 + 0.1 * torch.randn(shape, generator=g)
    if kind == 'norm_b':
        return 0.05 * torch.randn(shape, generator=g)
    if kind == 'bn_mean':
        return 0.1 * torch.randn(shape, generator=g)
    if kind == 'bn_var':
        return 0.8 + 0.4 * torch.rand(shape, generator=g)
    if kind == 'bn_count':
        return torch.zeros(shape, dtype=torch.int64)
    if kind == 'rpb_table':
        return 0.5 * torch.randn(shape, generator=g)
    if kind == 'rpb_index':
        idx = relative_position_index(WINDOW if window is None else tuple(window))
        assert tuple(idx.shape) == tuple(shape), (name, shape, window)
        return idx
    if kind == 'codebook':                       # nn.Embedding init N(0,1); padding row = 0
        w = torch.randn(shape, generator=g)
        w[-1].zero_()
        return w
    if kind == 'codebook_nopad':                 # VQGAN's nn.Embedding: N(0,1) init, no padding row
        return torch.randn(shape, generator=g)
    if kind == 'pos_emb':                        # non-zero (the reference initialises zeros, which hides indexing errors)
        return 0.5 * torch.randn(shape, generator=g)
    if kind == 'zeros':
        return torch.zeros(shape)
    raise ValueError(kind)


def synth_state_dict(spec, seed=0):
    sd = {}
    alias = getattr(spec, 'alias_of', lambda name: None)
    for name, (shape, kind, dtype) in spec.items():
        if kind == 'codebook_ema' or alias(name):
            continue
        sd[name] = synth_tensor(name, shape, kind, dtype, seed, window=getattr(spec, 'windows', {}).get(name))
    for name, (shape, kind, dtype) in spec.items():
        if kind == 'codebook_ema' and not alias(name):     # embed_ema = weight[:-1] clone (tdcrqvae3_arch.py:96)
            sd[name] = sd[name.replace('embed_ema', 'weight')][:-1].clone()
    for name in spec:
        if alias(name):                                    # a shared codebook: every depth's keys are one tensor
            sd[name] = sd[alias(name)]
    return {k: sd[k] for k in spec}
