"""TEST INFRASTRUCTURE ONLY — imports the *unmodified* reference (a read-only checkout of
kepengxu/PGTFormer at PGT_REFERENCE_ROOT) as a CPU oracle.  Never imported by product code or by the
tests.  Used to mint the committed golden vectors under tests/golden/ (see oracle/make_golden.py),
which pin oracle/pgt_oracle.py and the CUDA path against the real reference.

Recipe (SURVEY.md Appendix C):
  * two shim packages (oracle/shims/{basicsr,timm}) stand in for the absent imports
    (`archs/pgtformer_arch.py:15-16`, `archs/tdcrqvae3_arch.py:32`);
  * the reference is 512x512-only in three places (`archs/pgtformer_arch.py:375-378`, `:649`,
    `:535-550,698-700`); `generalise_size` applies the three run-time patches (bit-identical at
    512x512) so that fixtures at other sizes, H != W included, can be generated;
  * the reference crashes for clip-batch b>1 (`modules/rstt_layers.py:896-904`): callers loop
    over clips (b=1).
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get('PGT_REFERENCE_ROOT', '')     # a checkout of kepengxu/PGTFormer
_SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'shims')


def reference_available():
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, 'archs', 'pgtformer_arch.py'))


def _ensure_paths():
    for p in (_SHIMS, REFERENCE_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)


def import_reference():
    """Returns the reference's `archs.pgtformer_arch` module (imported from REFERENCE_ROOT)."""
    if not reference_available():
        raise RuntimeError('reference tree not present at %r (set PGT_REFERENCE_ROOT)' % REFERENCE_ROOT)
    _ensure_paths()
    # The product repo also has a top-level `archs` package (the drop-in). Make sure the name
    # `archs` resolves to the reference's while importing it, then restore.
    saved = {k: v for k, v in sys.modules.items() if k == 'archs' or k.startswith('archs.')
             or k == 'modules' or k.startswith('modules.')}
    for k in saved:
        del sys.modules[k]
    here_repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    saved_path = list(sys.path)
    sys.path = [p for p in sys.path if os.path.abspath(p or os.getcwd()) != here_repo]
    sys.path.insert(0, REFERENCE_ROOT)
    sys.path.insert(0, _SHIMS)
    cwd = os.getcwd()
    try:
        os.chdir(REFERENCE_ROOT)          # the files do sys.path.append(os.getcwd())
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            import archs.pgtformer_arch as ref_mod
        ref_pkg = {k: v for k, v in sys.modules.items() if k == 'archs' or k.startswith('archs.')
                   or k == 'modules' or k.startswith('modules.')}
    finally:
        os.chdir(cwd)
        sys.path = saved_path
    # park the reference packages under a private prefix and restore whatever was there before
    for k, v in ref_pkg.items():
        sys.modules['_pgt_reference.' + k] = v
        del sys.modules[k]
    sys.modules.update(saved)
    return ref_mod


def build_reference_model(network_g, state_dict=None, seed=0):
    """Constructs the reference PGTFormer (`archs/pgtformer_arch.py:490`) from a `network_g`
    option dict (`options/release_test_stage_IIII_dont_need_align_version.yml:53-90`)."""
    import contextlib
    import io
    import torch
    ref_mod = import_reference()
    opt = dict(network_g)
    opt.pop('type', None)
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        m = ref_mod.PGTFormer(**opt)
    m.eval()                                  # statement form: returns None (SURVEY F3)
    if state_dict is not None:
        m.load_state_dict(state_dict, strict=True)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def generalise_size(m, H, W):
    """Three run-time patches that lift the 512x512 restriction (SURVEY F4 / Appendix C step 4).
    Bit-identical to the unpatched model at 512x512.  H and W may differ: the fusion keys the reference looks up are
    feature widths (`feat.shape[-1]`), which the rescaled keys below follow."""
    import torch
    import torch.nn.functional as F
    assert H % 64 == 0 and W % 64 == 0
    cn = m.conditionnet

    def bisenet_forward(self, x):           # `archs/pgtformer_arch.py:365-379` with (32,32)->(H/16,W/16)
        Hh, Ww = x.size()[2:]
        feat_res8, feat_cp8, feat_cp16 = self.cp(x)
        feat_fuse = self.ffm(feat_res8, feat_cp8)
        feat_out = self.conv_out(feat_fuse)
        feat_out16 = self.conv_out16(feat_cp8)
        feat_out32 = self.conv_out32(feat_cp16)
        size = (Hh // 16, Ww // 16)
        feat_out = F.interpolate(feat_out, size, mode='bilinear', align_corners=True)
        feat_out16 = F.interpolate(feat_out16, size, mode='bilinear', align_corners=True)
        return torch.cat([feat_out, feat_out16, feat_out32], 1)

    cn.forward = types.MethodType(bisenet_forward, cn)
    m.quantizer.code_shape = torch.Size([H // 16, W // 16, 1])
    if not hasattr(m, '_pgt_orig_keys'):
        m._pgt_orig_keys = (list(m.connect_list), dict(m.fuse_encoder_indices))
        m._pgt_orig_fuse = {k: v for k, v in m.fuse_convs_dict.items()}
    conn, idx = m._pgt_orig_keys
    scale = lambda k: str(int(k) * W // 512)
    m.connect_list = [scale(k) for k in conn]
    m.fuse_encoder_indices = {scale(k): v for k, v in idx.items()}
    # plain dict view keyed by the rescaled widths (forward only does [] lookup)
    m.__dict__['_modules']['fuse_convs_dict'] = torch.nn.ModuleDict(
        {scale(k): v for k, v in m._pgt_orig_fuse.items()})
    return m


def reference_forward(m, x, w=1.0, adain=True, code_only=None):
    """Runs the reference one clip (3 frames) at a time and concatenates (SURVEY F5)."""
    import torch
    t = m.t
    assert x.shape[0] % t == 0
    outs = []
    with torch.no_grad():
        for i in range(x.shape[0] // t):
            generalise_size(m, x.shape[2], x.shape[3])
            outs.append(m(x[i * t:(i + 1) * t], w=w, adain=adain, code_only=code_only))
    return tuple(torch.cat([o[j] for o in outs], 0) for j in range(len(outs[0])))
