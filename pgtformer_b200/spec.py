"""State-dict layout of PGTFormer (names, shapes, kinds) derived from a `network_g` option dict.

The drop-in must load the reference's checkpoints with `strict=True` (SURVEY App. D), so the
parameter/buffer names below are the reference's: they follow the module attribute names of
`archs/pgtformer_arch.py:491-556` (PGTFormer ctor), `archs/tdcrqvae3_arch.py:460-539,577-670`
(Encoder/Decoder ctor), `modules/rstt_layers.py:134-193,236-282,499-533,835-873` (window
attention / Swin block / EncoderLayer / TDResnetBlock ctors), `archs/codeformer_arch.py:102-117`
(TransformerSALayer) and `archs/pgtformer_arch.py:34-397` (BiSeNet / ResNet18).

`kind` drives the deterministic synthetic initialisation in weights.py and the kernel-layout
repack in engine.py.
"""
from collections import OrderedDict

WINDOW = (3, 4, 4)            # frames x Wh x Ww  (num_frames=3, window_sizes=[4,4])
N_WIN_TOK = 48


class Spec(OrderedDict):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.windows = {}         # name of a relative_position_index buffer -> its (D, H, W) window (default: WINDOW)
        # module prefix -> the module it is: a shared codebook is one VQEmbedding listed under every depth
        # (`archs/tdcrqvae3_arch.py:256-262`), so its state-dict keys repeat once per depth, all aliasing one tensor
        self.module_aliases = {}

    def alias_of(self, name):
        """The key whose tensor `name` aliases, or None."""
        mod, _, leaf = name.rpartition('.')
        return self.module_aliases[mod] + '.' + leaf if mod in self.module_aliases else None

    def add(self, name, shape, kind, dtype='float32'):
        assert name not in self, name
        self[name] = (tuple(int(s) for s in shape), kind, dtype)


def _conv(s, p, cin, cout, k, bias=True):
    s.add(p + '.weight', (cout, cin, k, k), 'conv_w')
    if bias:
        s.add(p + '.bias', (cout,), 'bias')


def _linear(s, p, cin, cout, bias=True):
    s.add(p + '.weight', (cout, cin), 'linear_w')
    if bias:
        s.add(p + '.bias', (cout,), 'bias')


def _norm(s, p, c):
    s.add(p + '.weight', (c,), 'norm_w')
    s.add(p + '.bias', (c,), 'norm_b')


def _bn(s, p, c):
    s.add(p + '.weight', (c,), 'norm_w')
    s.add(p + '.bias', (c,), 'norm_b')
    s.add(p + '.running_mean', (c,), 'bn_mean')
    s.add(p + '.running_var', (c,), 'bn_var')
    s.add(p + '.num_batches_tracked', (), 'bn_count', 'int64')


def _td_resblock(s, p, cin, cout):
    _norm(s, p + '.norm1', cin)
    _conv(s, p + '.conv1', cin, cout, 3)
    _norm(s, p + '.norm2', cout)
    _conv(s, p + '.conv2', cout, cout, 3)
    if cin != cout:
        _conv(s, p + '.nin_shortcut', cin, cout, 1)


def _swin_block(s, p, c, heads):
    d, wh, ww = WINDOW
    _norm(s, p + '.norm1', c)
    s.add(p + '.attn.relative_position_bias_table', ((2 * d - 1) * (2 * wh - 1) * (2 * ww - 1), heads), 'rpb_table')
    s.add(p + '.attn.relative_position_index', (N_WIN_TOK, N_WIN_TOK), 'rpb_index', 'int64')
    _linear(s, p + '.attn.q', c, c)
    _linear(s, p + '.attn.kv', c, 2 * c)
    _linear(s, p + '.attn.proj', c, c)
    _norm(s, p + '.norm2', c)
    _linear(s, p + '.mlp.fc1', c, c)          # mlp_ratio = 1
    _linear(s, p + '.mlp.fc2', c, c)


def _encoder_layer(s, p, c, depth, heads):
    for i in range(depth):
        _swin_block(s, '%s.blocks.%d' % (p, i), c, heads)


def _convbnrelu(s, p, cin, cout, k):
    _conv(s, p + '.conv', cin, cout, k, bias=False)
    _bn(s, p + '.bn', cout)


def _basic_block(s, p, cin, cout, stride):
    _conv(s, p + '.conv1', cin, cout, 3, bias=False)
    _bn(s, p + '.bn1', cout)
    _conv(s, p + '.conv2', cout, cout, 3, bias=False)
    _bn(s, p + '.bn2', cout)
    if cin != cout or stride != 1:
        _conv(s, p + '.downsample.0', cin, cout, 1, bias=False)
        _bn(s, p + '.downsample.1', cout)


def _bisenet(s, p, n_classes=19):
    r = p + '.cp.resnet'
    _conv(s, r + '.conv1', 3, 64, 7, bias=False)
    _bn(s, r + '.bn1', 64)
    for li, (cin, cout, stride) in enumerate([(64, 64, 1), (64, 128, 2), (128, 256, 2), (256, 512, 2)], 1):
        _basic_block(s, '%s.layer%d.0' % (r, li), cin, cout, stride)
        _basic_block(s, '%s.layer%d.1' % (r, li), cout, cout, 1)
    for name, cin in (('arm16', 256), ('arm32', 512)):
        _convbnrelu(s, '%s.cp.%s.conv' % (p, name), cin, 128, 3)
        _conv(s, '%s.cp.%s.conv_atten' % (p, name), 128, 128, 1, bias=False)
        _bn(s, '%s.cp.%s.bn_atten' % (p, name), 128)
    _convbnrelu(s, p + '.cp.conv_head32', 128, 128, 3)
    _convbnrelu(s, p + '.cp.conv_head16', 128, 128, 3)
    _convbnrelu(s, p + '.cp.conv_avg', 512, 128, 1)
    _convbnrelu(s, p + '.ffm.convblk', 256, 256, 1)
    _conv(s, p + '.ffm.conv1', 256, 64, 1, bias=False)
    _conv(s, p + '.ffm.conv2', 64, 256, 1, bias=False)
    for name, cin, mid in (('conv_out', 256, 256), ('conv_out16', 128, 64), ('conv_out32', 128, 64)):
        _convbnrelu(s, '%s.%s.conv' % (p, name), cin, mid, 3)
        _conv(s, '%s.%s.conv_out' % (p, name), mid, n_classes, 1, bias=False)


class Arch:
    """Resolved architecture constants (everything the engine / oracle need besides weights)."""

    def __init__(self, network_g):
        g = dict(network_g)
        dd = dict(g['ddconfig'])
        self.tf = int(g.get('tf', 3))
        self.embed_dim = int(g.get('embed_dim', 64))
        self.n_embed = int(g.get('n_embed', 512))
        self.code_shape = tuple(g['code_shape'])
        self.latent_shape = tuple(g['latent_shape'])
        self.shared_codebook = bool(g.get('shared_codebook', True))       # the options files' setting
        self.dim_embd = int(g.get('dim_embd', 512))
        self.n_head = int(g.get('n_head', 8))
        self.n_layers = int(g.get('n_layers', 9))
        self.connect_list = list(g.get('connect_list', ['32', '64', '128', '256']))
        self.ch = int(dd['ch'])
        self.ch_mult = tuple(dd['ch_mult'])
        self.num_res_blocks = int(dd['num_res_blocks'])
        self.depths = tuple(dd['depths'])
        self.num_heads = tuple(dd['num_heads'])
        self.num_frames = int(dd['num_frames'])
        self.window_sizes = tuple(tuple(w) for w in dd['window_sizes'])
        self.resolution = int(dd['resolution'])
        self.attn_resolutions = tuple(dd['attn_resolutions'])
        self.z_channels = int(dd['z_channels'])
        self.in_channels = int(dd['in_channels'])
        self.out_ch = int(dd['out_ch'])
        self.double_z = bool(dd.get('double_z', True))
        self.num_levels = len(self.ch_mult)
        if g.get('bottleneck_type', 'rq') != 'rq':
            raise ValueError("invalid 'bottleneck_type' (must be 'rq')")     # tdcrqvae3_arch.py:752
        if not len(self.code_shape) == len(self.latent_shape) == 3:
            raise ValueError('incompatible code shape or latent shape')      # tdcrqvae3_arch.py:232
        if any(y % x != 0 for x, y in zip(self.code_shape[:2], self.latent_shape[:2])):
            raise ValueError('incompatible code shape or latent shape')      # tdcrqvae3_arch.py:234
        if self.tf != 3 or self.num_frames != 3 or any(w != (4, 4) for w in self.window_sizes):
            raise ValueError('the CUDA path is built for 3-frame clips and 4x4x3 windows')
        if int(self.code_shape[2]) < 1:
            raise ValueError('quantiser depth code_shape[2] must be >= 1, got %r' % (self.code_shape[2],))
        self.depth = int(self.code_shape[2])
        # levels that carry a window-attention layer (curr_res walk of tdcrqvae3_arch.py:482-510)
        self.level_has_attn = tuple((self.resolution >> i) in self.attn_resolutions
                                    for i in range(self.num_levels))
        self.level_ch = tuple(self.ch * m for m in self.ch_mult)
        # SFT fusion after decoder level i <-> key str(resolution >> i)  (pgtformer_arch.py:535-550)
        self.fuse_level_key = {i: str(self.resolution >> i) for i in range(self.num_levels)
                               if str(self.resolution >> i) in self.connect_list}
        self.fuse_channels = {'16': 512, '32': 512, '64': 256, '128': 256, '256': 128, '512': 64}


def build_spec(network_g):
    a = Arch(network_g)
    s = Spec()
    in_mult = (1,) + a.ch_mult
    # ---- encoder (tdcrqvae3_arch.py:460-539)
    _conv(s, 'encoder.conv_in', a.in_channels, a.ch, 3)
    block_in = a.ch
    for lvl in range(a.num_levels):
        block_in = a.ch * in_mult[lvl]
        block_out = a.ch * a.ch_mult[lvl]
        for b in range(a.num_res_blocks):
            _td_resblock(s, 'encoder.down.%d.block.%d' % (lvl, b), block_in, block_out)
            block_in = block_out
            if a.level_has_attn[lvl]:
                _encoder_layer(s, 'encoder.down.%d.attn.%d' % (lvl, b), block_in, a.depths[lvl], a.num_heads[lvl])
        if lvl != a.num_levels - 1:
            _conv(s, 'encoder.down.%d.downsample.conv' % lvl, block_in, block_in, 3)
    _td_resblock(s, 'encoder.mid.block_1', block_in, block_in)
    _encoder_layer(s, 'encoder.mid.attn_1', block_in, a.depths[-1], a.num_heads[-1])
    _td_resblock(s, 'encoder.mid.block_2', block_in, block_in)
    _norm(s, 'encoder.norm_out', block_in)
    _conv(s, 'encoder.conv_out', block_in, 2 * a.z_channels if a.double_z else a.z_channels, 3)
    # ---- decoder (tdcrqvae3_arch.py:577-670)
    block_in = a.ch * a.ch_mult[-1]
    _conv(s, 'decoder.conv_in', a.z_channels, block_in, 3)
    _td_resblock(s, 'decoder.mid.block_1', block_in, block_in)
    _encoder_layer(s, 'decoder.mid.attn_1', block_in, a.depths[-1], a.num_heads[-1])
    _td_resblock(s, 'decoder.mid.block_2', block_in, block_in)
    for lvl in reversed(range(a.num_levels)):
        block_out = a.ch * a.ch_mult[lvl]
        for b in range(a.num_res_blocks + 1):
            _td_resblock(s, 'decoder.up.%d.block.%d' % (lvl, b), block_in, block_out)
            block_in = block_out
            if a.level_has_attn[lvl]:
                _encoder_layer(s, 'decoder.up.%d.attn.%d' % (lvl, b), block_in, a.depths[lvl], a.num_heads[lvl])
        if lvl != 0:
            _conv(s, 'decoder.up.%d.upsample.conv' % lvl, block_in, block_in, 3)
    _norm(s, 'decoder.norm_out', block_in)
    _conv(s, 'decoder.conv_out', block_in, a.out_ch, 3)
    # ---- quantiser (tdcrqvae3_arch.py:80-97,215-271): one VQEmbedding per depth, or one shared by every depth
    e = a.embed_dim
    for d in range(a.depth):
        p = 'quantizer.codebooks.%d' % d
        s.add(p + '.weight', (a.n_embed + 1, e), 'codebook')
        s.add(p + '.cluster_size_ema', (a.n_embed,), 'zeros')
        s.add(p + '.embed_ema', (a.n_embed, e), 'codebook_ema')
        if a.shared_codebook and d > 0:
            s.module_aliases[p] = 'quantizer.codebooks.0'
    _conv(s, 'quant_conv', a.z_channels, e, 1)
    _conv(s, 'post_quant_conv', e, a.z_channels, 1)
    # ---- PGTFormer head (pgtformer_arch.py:511-550)
    _bisenet(s, 'conditionnet')
    _conv(s, 'convpos', 57, 512, 1)
    _linear(s, 'feat_emb', 512, a.dim_embd)
    for i in range(a.n_layers):
        p = 'ft_layers.%d' % i
        s.add(p + '.self_attn.in_proj_weight', (3 * a.dim_embd, a.dim_embd), 'linear_w')
        s.add(p + '.self_attn.in_proj_bias', (3 * a.dim_embd,), 'bias')
        _linear(s, p + '.self_attn.out_proj', a.dim_embd, a.dim_embd)
        _linear(s, p + '.linear1', a.dim_embd, 2 * a.dim_embd)
        _linear(s, p + '.linear2', 2 * a.dim_embd, a.dim_embd)
        _norm(s, p + '.norm1', a.dim_embd)
        _norm(s, p + '.norm2', a.dim_embd)
    _norm(s, 'idx_pred_layer.0', a.dim_embd)
    _linear(s, 'idx_pred_layer.1', a.dim_embd, a.code_shape[2] * a.n_embed, bias=False)
    for key in a.connect_list:
        c = a.fuse_channels[key]
        p = 'fuse_convs_dict.' + key
        tcc, t = 32, a.tf
        _norm(s, p + '.encode_enc.norm1', 2 * c + tcc)
        _conv(s, p + '.encode_enc.conv1', 2 * c + tcc, c, 3)
        _norm(s, p + '.encode_enc.norm2', c)
        _conv(s, p + '.encode_enc.conv2', c, c, 3)
        _conv(s, p + '.encode_enc.conv_out', 2 * c + tcc, c, 1)
        for br in ('scale', 'shift'):
            _conv(s, '%s.%s.0' % (p, br), c, c, 3)
            _conv(s, '%s.%s.2' % (p, br), c, c, 3)
        _conv(s, p + '.tconvenc', c, tcc, 1)
        _conv(s, p + '.tconvdec', c, tcc, 1)
        _conv(s, p + '.tfusion0', 2 * t * tcc, tcc * t, 1)
        _conv(s, p + '.tfusion1', tcc, tcc, 1)
    return a, s


# --------------------------------------------------------------------------- TDRQVAE (archs/tdrqvae_arch.py:787-841)
ATTN_WIDTHS = (64, 256, 512)          # pgt_mha_fwd head widths (the AttnBlock is one head of width C)
SWIN_HEAD_WIDTHS = (16, 32, 64)       # pgt_window3d_attention head widths
SWIN_MAX_TOKENS = 128                 # pgt_window3d_attention: tokens per window


def _attn_block(s, p, c):
    """AttnBlock (`archs/tdrqvae_arch.py:151-176`): GroupNorm + four 1x1 convs."""
    _norm(s, p + '.norm', c)
    for n in ('q', 'k', 'v', 'proj_out'):
        _conv(s, '%s.%s' % (p, n), c, c, 1)


def _swin3d_layer(s, p, c, depth, heads, window, mlp_ratio=4):
    """Video-Swin BasicLayer (`modules/swin.py:326-378`): depth x SwinTransformerBlock3D, qkv without bias."""
    n = window[0] * window[1] * window[2]
    nrel = (2 * window[0] - 1) * (2 * window[1] - 1) * (2 * window[2] - 1)
    for i in range(depth):
        b = '%s.blocks.%d' % (p, i)
        _norm(s, b + '.norm1', c)
        s.add(b + '.attn.relative_position_bias_table', (nrel, heads), 'rpb_table')
        s.add(b + '.attn.relative_position_index', (n, n), 'rpb_index', 'int64')
        s.windows[b + '.attn.relative_position_index'] = tuple(window)
        _linear(s, b + '.attn.qkv', c, 3 * c, bias=False)
        _linear(s, b + '.attn.proj', c, c)
        _norm(s, b + '.norm2', c)
        _linear(s, b + '.mlp.fc1', c, mlp_ratio * c)
        _linear(s, b + '.mlp.fc2', mlp_ratio * c, c)


class TDRQVAEArch:
    """Resolved constants of TDRQVAE: the 2-D RQ-VAE Encoder / Decoder (`archs/tdrqvae_arch.py:587-784`) around a
    depth-1 RQBottleneck and two Video-Swin BasicLayers.  Raises ValueError for what the reference rejects and for
    what the CUDA kernels cannot run."""

    def __init__(self, network_g):
        g = dict(network_g)
        dd = dict(g['ddconfig'])
        self.tf = int(g.get('tf', 7))
        self.embed_dim = int(g.get('embed_dim', 64))
        self.n_embed = int(g.get('n_embed', 512))
        if g.get('bottleneck_type', 'rq') != 'rq':
            raise ValueError("invalid 'bottleneck_type' (must be 'rq')")     # tdrqvae_arch.py:829
        self.latent_shape = tuple(g['latent_shape'])
        self.code_shape = tuple(g['code_shape'])
        if not len(self.code_shape) == len(self.latent_shape) == 3:
            raise ValueError('incompatible code shape or latent shape')      # tdrqvae_arch.py:357-360
        if any(y % x != 0 for x, y in zip(self.code_shape[:2], self.latent_shape[:2])):
            raise ValueError('incompatible code shape or latent shape')
        if self.code_shape[2] != 1:
            # the reference's TDRQVAE.forward / get_codes reshape the codes with code.view(b, t, fh, fw, 1)
            # (archs/tdrqvae_arch.py:852, 888), which fails for any deeper quantiser
            raise ValueError('TDRQVAE runs quantiser depth 1 only: the reference reshapes its codes with '
                             'view(b, t, h, w, 1) (archs/tdrqvae_arch.py:852, 888)')
        self.ch = int(dd['ch'])
        self.ch_mult = tuple(dd['ch_mult'])
        self.num_res_blocks = int(dd['num_res_blocks'])
        self.resolution = int(dd['resolution'])
        self.attn_resolutions = tuple(dd['attn_resolutions'])
        self.z_channels = int(dd['z_channels'])
        self.in_channels = int(dd['in_channels'])
        self.out_ch = int(dd['out_ch'])
        self.double_z = bool(dd.get('double_z', True))
        self.stages_atten = int(dd['stages_atten'])
        self.num_head = int(dd['num_head'])
        self.window_size = tuple(int(w) for w in dd['window_size'])
        self.num_levels = len(self.ch_mult)
        self.down = 2 ** (self.num_levels - 1)                            # frame size / latent size
        self.level_ch = tuple(self.ch * m for m in self.ch_mult)
        # levels with AttnBlocks: the curr_res walk of the constructor (:606-627), fixed by `resolution`
        self.level_has_attn = tuple((self.resolution >> i) in self.attn_resolutions for i in range(self.num_levels))
        if self.double_z:
            raise ValueError('double_z: Encoder.conv_out would give 2 * z_channels, quant_conv reads z_channels')
        if self.in_channels != 3 or self.ch != 64:
            raise ValueError('the CUDA path is built for RGB input and ch = 64')
        if any(c % 32 for c in self.level_ch):
            raise ValueError('GroupNorm(32): every level width must be a multiple of 32')
        widths = {c for c, a in zip(self.level_ch, self.level_has_attn) if a} | {self.level_ch[-1]}
        if not widths <= set(ATTN_WIDTHS):
            raise ValueError('AttnBlock widths %s: the attention kernel takes %s' % (sorted(widths), ATTN_WIDTHS))
        if self.stages_atten < 1 or self.num_head < 1 or self.embed_dim % self.num_head or \
                self.embed_dim // self.num_head not in SWIN_HEAD_WIDTHS:
            raise ValueError('Video-Swin layers of %d blocks, %d heads over %d channels: head width must be one of %s'
                             % (self.stages_atten, self.num_head, self.embed_dim, SWIN_HEAD_WIDTHS))
        if len(self.window_size) != 3 or min(self.window_size) < 1 or \
                self.window_size[0] * self.window_size[1] * self.window_size[2] > SWIN_MAX_TOKENS:
            raise ValueError('Video-Swin window %s: at most %d tokens' % (self.window_size, SWIN_MAX_TOKENS))


def build_tdrqvae_spec(network_g):
    a = TDRQVAEArch(network_g)
    s = Spec()
    in_mult = (1,) + a.ch_mult
    # ---- Encoder (tdrqvae_arch.py:587-648)
    _conv(s, 'encoder.conv_in', a.in_channels, a.ch, 3)
    for lvl in range(a.num_levels):
        block_in = a.ch * in_mult[lvl]
        block_out = a.level_ch[lvl]
        for b in range(a.num_res_blocks):
            _td_resblock(s, 'encoder.down.%d.block.%d' % (lvl, b), block_in, block_out)
            block_in = block_out
        if a.level_has_attn[lvl]:
            for b in range(a.num_res_blocks):
                _attn_block(s, 'encoder.down.%d.attn.%d' % (lvl, b), block_in)
        if lvl != a.num_levels - 1:
            _conv(s, 'encoder.down.%d.downsample.conv' % lvl, block_in, block_in, 3)
    _td_resblock(s, 'encoder.mid.block_1', block_in, block_in)
    _attn_block(s, 'encoder.mid.attn_1', block_in)
    _td_resblock(s, 'encoder.mid.block_2', block_in, block_in)
    _norm(s, 'encoder.norm_out', block_in)
    _conv(s, 'encoder.conv_out', block_in, a.z_channels, 3)
    # ---- Decoder (:683-751)
    block_in = a.level_ch[-1]
    _conv(s, 'decoder.conv_in', a.z_channels, block_in, 3)
    _td_resblock(s, 'decoder.mid.block_1', block_in, block_in)
    _attn_block(s, 'decoder.mid.attn_1', block_in)
    _td_resblock(s, 'decoder.mid.block_2', block_in, block_in)
    for lvl in reversed(range(a.num_levels)):
        block_out = a.level_ch[lvl]
        for b in range(a.num_res_blocks + 1):
            _td_resblock(s, 'decoder.up.%d.block.%d' % (lvl, b), block_in, block_out)
            block_in = block_out
        if a.level_has_attn[lvl]:
            for b in range(a.num_res_blocks + 1):
                _attn_block(s, 'decoder.up.%d.attn.%d' % (lvl, b), block_in)
        if lvl != 0:
            _conv(s, 'decoder.up.%d.upsample.conv' % lvl, block_in, block_in, 3)
    _norm(s, 'decoder.norm_out', block_in)
    _conv(s, 'decoder.conv_out', block_in, a.out_ch, 3)
    # ---- quantiser (:206-223, 381-394): one shared codebook of depth 1
    e = a.embed_dim
    s.add('quantizer.codebooks.0.weight', (a.n_embed + 1, e), 'codebook')
    s.add('quantizer.codebooks.0.cluster_size_ema', (a.n_embed,), 'zeros')
    s.add('quantizer.codebooks.0.embed_ema', (a.n_embed, e), 'codebook_ema')
    _conv(s, 'quant_conv', a.z_channels, e, 1)
    _conv(s, 'post_quant_conv', e, a.z_channels, 1)
    for p in ('tdswin_pre', 'tdswin_post'):
        _swin3d_layer(s, p, e, a.stages_atten, a.num_head, a.window_size)
    return a, s
