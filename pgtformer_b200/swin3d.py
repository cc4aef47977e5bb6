"""Video-Swin `BasicLayer` (SURVEY 8(f) #4, second half) on the H100 kernels: depth x SwinTransformerBlock3D
(`modules/swin.py:170-271` of the reference) = LayerNorm -> qkv projection -> 3-D shifted-window attention with zero
padding to window multiples (pgt_window3d_attention) -> proj + residual -> LayerNorm -> Mlp (ratio 4, exact GELU) +
residual.  Activations are channels-last bf16 token rows [B*D*H*W, C]; every op is a call into libpgt_b200.so."""
import torch
import torch.nn as nn

BF = torch.bfloat16


def _rel_index(window):
    cd, ch, cw = (torch.arange(n) for n in window)
    coords = torch.stack(torch.meshgrid(cd, ch, cw, indexing='ij')).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += window[0] - 1
    rel[:, :, 1] += window[1] - 1
    rel[:, :, 2] += window[2] - 1
    rel[:, :, 0] *= (2 * window[1] - 1) * (2 * window[2] - 1)
    rel[:, :, 1] *= 2 * window[2] - 1
    return rel.sum(-1)


class _Holder(nn.Module):
    pass


class BasicLayer(nn.Module):
    def __init__(self, dim, depth, num_heads, window_size=(1, 7, 7), mlp_ratio=4., qkv_bias=False, qk_scale=None,
                 drop=0., attn_drop=0., drop_path=0., norm_layer=nn.LayerNorm, downsample=None, use_checkpoint=False):
        super().__init__()
        if downsample is not None or qk_scale is not None:
            raise ValueError('pgtformer_b200 BasicLayer: downsample / qk_scale are not used by TDRQVAE and not supported')
        self.dim, self.depth, self.num_heads = dim, depth, num_heads
        self.window_size = tuple(window_size)
        self.shift_size = tuple(i // 2 for i in self.window_size)
        hidden = int(dim * mlp_ratio)
        nrel = (2 * window_size[0] - 1) * (2 * window_size[1] - 1) * (2 * window_size[2] - 1)
        self.blocks = nn.ModuleList()
        for _ in range(depth):                       # the module tree only gives the parameters their reference names
            blk = _Holder()
            blk.norm1 = nn.LayerNorm(dim)
            blk.attn = _Holder()
            blk.attn.relative_position_bias_table = nn.Parameter(torch.zeros(nrel, num_heads))
            blk.attn.register_buffer('relative_position_index', _rel_index(self.window_size))
            blk.attn.qkv = nn.Linear(dim, 3 * dim, bias=qkv_bias)
            blk.attn.proj = nn.Linear(dim, dim)
            blk.norm2 = nn.LayerNorm(dim)
            blk.mlp = _Holder()
            blk.mlp.fc1 = nn.Linear(dim, hidden)
            blk.mlp.fc2 = nn.Linear(hidden, dim)
            nn.init.trunc_normal_(blk.attn.relative_position_bias_table, std=.02)
            self.blocks.append(blk)
        self.requires_grad_(False)
        self._packed = None

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._packed = None
        return r

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self._packed = None
        return r

    def _pack(self):
        if self._packed is None:
            named = dict(self.named_parameters())
            named.update(self.named_buffers())
            self._packed = pack_blocks(named.get, self.depth)
        return self._packed

    @torch.no_grad()
    def forward(self, x):
        """x: [B, C, D, H, W] on a CUDA device -> same shape and dtype (`modules/swin.py:380-405`)."""
        if not x.is_cuda:
            raise RuntimeError('pgtformer_b200 has no CPU path: BasicLayer needs a CUDA (sm_90a) device')
        B, C, D, H, W = x.shape
        heads = self.num_heads
        T = B * D * H * W
        with torch.cuda.device(x.device):
            h = x.permute(0, 2, 3, 4, 1).reshape(T, C).to(BF).contiguous()           # 'b c d h w -> b d h w c'
            h = basic_layer_rows(h, B, D, H, W, self._pack(), heads, self.window_size)
            return h.view(B, D, H, W, C).permute(0, 4, 1, 2, 3).to(x.dtype).contiguous()


def pack_blocks(get, depth):
    """Kernel-layout weights of `depth` SwinTransformerBlock3D; get('blocks.<i>.<name>') returns the reference-named
    tensor on the device (None for a qkv bias the layer does not have).  The expanded relative-position bias is
    cached per window size N in each block's 'bias' dict by basic_layer_rows."""
    w = []
    for i in range(depth):
        g = lambda n: get('blocks.%d.%s' % (i, n))
        qkv_b = g('attn.qkv.bias')
        d = {'n1w': g('norm1.weight').float().contiguous(), 'n1b': g('norm1.bias').float().contiguous(),
             'n2w': g('norm2.weight').float().contiguous(), 'n2b': g('norm2.bias').float().contiguous(),
             'qkv': g('attn.qkv.weight').to(BF).contiguous(),
             'qkv_b': qkv_b.float().contiguous() if qkv_b is not None else None,
             'proj': g('attn.proj.weight').to(BF).contiguous(), 'proj_b': g('attn.proj.bias').float().contiguous(),
             'fc1': g('mlp.fc1.weight').to(BF).contiguous(), 'fc1_b': g('mlp.fc1.bias').float().contiguous(),
             'fc2': g('mlp.fc2.weight').to(BF).contiguous(), 'fc2_b': g('mlp.fc2.bias').float().contiguous(),
             'table': g('attn.relative_position_bias_table').float(), 'index': g('attn.relative_position_index'),
             'bias': {}}
        # a padded token is a zero row after the norm: its projection is the qkv bias (or zero)
        d['pad'] = d['qkv_b'].to(BF).contiguous() if d['qkv_b'] is not None else None
        w.append(d)
    return w


def basic_layer_rows(h, B, D, H, W, blocks, heads, window, out=None):
    """BasicLayer.forward (`modules/swin.py:380-405`) on token rows: h [B*D*H*W, C] bf16 in (b, d, h, w) order (the
    'b d h w c' layout of the reference), blocks from pack_blocks.  Returns the rows after the last block: a new bf16
    tensor, or `out` (bf16 or fp32 [T, C]) when given, which the last block's fc2 + residual epilogue writes."""
    from . import ops
    T, C = h.shape
    shift_size = tuple(i // 2 for i in window)
    ws = tuple(min(s, w) for s, w in zip((D, H, W), window))                  # get_window_size
    N = ws[0] * ws[1] * ws[2]
    new = lambda *s, dt=BF: torch.empty(*s, dtype=dt, device=h.device)
    for i, d in enumerate(blocks):
        if N not in d['bias']:                                                 # relative_position_index[:N, :N]
            idx = d['index'][:N, :N].reshape(-1).to(h.device)
            d['bias'][N] = d['table'][idx].view(N, N, heads).permute(2, 0, 1).contiguous()
        shift = (0, 0, 0) if i % 2 == 0 else shift_size
        y = ops.layernorm(h, d['n1w'], d['n1b'], new(T, C))
        qkv = ops.linear(y, d['qkv'], new(T, 3 * C), bias=d['qkv_b'])
        a = ops.window3d_attention(qkv, B, D, H, W, C, heads, window, shift, d['bias'][N], new(T, C),
                                   pad_qkv=d['pad'])
        h = ops.linear(a, d['proj'], new(T, C), bias=d['proj_b'], residual=h)
        y = ops.layernorm(h, d['n2w'], d['n2b'], new(T, C))
        m = ops.linear(y, d['fc1'], new(T, d['fc1'].shape[0]), bias=d['fc1_b'], act=ops.ACT_GELU)
        last = out is not None and i == len(blocks) - 1
        h = ops.linear(m, d['fc2'], out if last else new(T, C), bias=d['fc2_b'], residual=h)
    return h
