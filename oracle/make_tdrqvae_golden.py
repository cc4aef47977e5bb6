"""TEST INFRASTRUCTURE ONLY — mints tests/golden/tdrqvae_*.pt and tests/golden/tdrqvae_state_dict_spec.json from the
UNMODIFIED reference's `archs/tdrqvae_arch.py` (imported with the basicsr / timm / mmcv shims of oracle/shims), built
from this repo's `network_g` with `type: TDRQVAE` and loaded with the deterministic synthetic checkpoint
(pgtformer_b200.weights.synth_state_dict of build_tdrqvae_spec, seed 0) with strict=True:

    PGT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_tdrqvae_golden

The reference's TDRQVAE runs any b and t.  forward and get_codes need no size patch; decode_code away from 512^2 needs
the `quantizer.code_shape` patch of reference_loader.generalise_size (applied here alone: TDRQVAE has no parsing net).

Fixtures (inputs are not stored: `golden_clips(seed, b, t, H, W)` regenerates them bit-exactly):
  64^2,  b = 1, t = 3: whole tensors;
  128^2, b = 2, t = 7: the depth is padded 7 -> 10 and the windows are shifted in depth; strided samples;
  64x192, b = 1, t = 3: H != W; strided samples;
  512^2, b = 1, t = 3: the reference's native size, compact: frame samples as fp16 (the reference materialises
  [F, 16384, 16384] fp32 scores at its 128^2 AttnBlocks, so F stays 3).
Each records z_e = encode(frames), the same after tdswin_pre, every code with its top-2 distance margin, quant_loss, the
code_only z_q, out, decode_code of the reference's own codes and a soft-code sample (temp 1)."""
import contextlib
import io
import json
import os
import sys
import time

import torch

from oracle.make_golden import GOLDEN, load_network_g, sample_into

SPEC_JSON = os.path.join(GOLDEN, 'tdrqvae_state_dict_spec.json')
# (seed, b, t, H[, W]) -> flat sample strides of the large tensors; None keeps the tensor whole
CASES = {(31, 1, 3, 64): None,
         (32, 2, 7, 128): {'z': 16, 'out': 32, 'soft': 64},
         (33, 1, 3, 512): {'z': 64, 'out': 64, 'soft': 256},
         (34, 1, 3, 64, 192): {'z': 4, 'out': 4, 'soft': 16}}


def network_g():
    g = dict(load_network_g())
    g['type'] = 'TDRQVAE'
    return g


def golden_clips(seed, b, t, H, W=None):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, t, 3, H, H if W is None else W, generator=g)


def golden_name(seed, b, t, H, W=None):
    size = '%d' % H if W is None else '%dx%d' % (H, W)
    return 'tdrqvae_ref_b%d_t%d_%s_seed%d.pt' % (b, t, size, seed)


def import_reference_tdrqvae():
    """The reference's `archs.tdrqvae_arch` module, imported from PGT_REFERENCE_ROOT as oracle/reference_loader.py
    imports `archs.pgtformer_arch`: the names `archs` / `modules` resolve to the reference's while importing, and the
    repo's own packages are restored afterwards."""
    from oracle.reference_loader import REFERENCE_ROOT, _SHIMS, reference_available
    if not reference_available():
        raise RuntimeError('reference tree not present at %r (set PGT_REFERENCE_ROOT)' % REFERENCE_ROOT)
    own = lambda k: k in ('archs', 'modules') or k.startswith(('archs.', 'modules.'))
    saved = {k: v for k, v in sys.modules.items() if own(k)}
    for k in saved:
        del sys.modules[k]
    here_repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    saved_path = list(sys.path)
    sys.path = [p for p in sys.path if os.path.abspath(p or os.getcwd()) != here_repo]
    sys.path.insert(0, REFERENCE_ROOT)
    sys.path.insert(0, _SHIMS)
    cwd = os.getcwd()
    try:
        os.chdir(REFERENCE_ROOT)          # the file does sys.path.append(os.getcwd())
        with contextlib.redirect_stdout(io.StringIO()):
            import archs.tdrqvae_arch as ref_mod
        ref_pkg = {k: v for k, v in sys.modules.items() if own(k)}
    finally:
        os.chdir(cwd)
        sys.path = saved_path
    for k, v in ref_pkg.items():
        sys.modules['_pgt_reference_tdrqvae.' + k] = v
        del sys.modules[k]
    sys.modules.update(saved)
    return ref_mod


def reference_model():
    from pgtformer_b200.spec import build_tdrqvae_spec
    from pgtformer_b200.weights import synth_state_dict
    ref_mod = import_reference_tdrqvae()
    g = network_g()
    _, spec = build_tdrqvae_spec(g)
    opt = dict(g)
    opt.pop('type')
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = ref_mod.TDRQVAE(**opt)
    m.eval()
    m.load_state_dict(synth_state_dict(spec, 0), strict=True)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def write_spec(m):
    spec = {k: [list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()}
    with open(SPEC_JSON, 'w') as f:
        json.dump(spec, f, indent=0, sort_keys=False)
        f.write('\n')
    print('wrote %s (%d entries)' % (SPEC_JSON, len(spec)))


def mint(m, seed, b, t, H, strides, W=None):
    x = golden_clips(seed, b, t, H, W)
    W = H if W is None else W
    Fr, h, w = b * t, H // 16, W // 16
    m.quantizer.code_shape = torch.Size([h, w, 1])           # generalise_size's patch (decode_code only)
    t0 = time.time()
    with torch.no_grad():
        out, loss, code = m(x)
        z_q, loss2, code2 = m(x, code_only=True)
        assert torch.equal(code, code2) and torch.equal(loss, loss2)
        z_e = m.encode(x.view(Fr, 3, H, W))
        z_pre = m.tdswin_pre(z_e.view(b, t, h, w, -1).permute(0, 4, 1, 2, 3)).permute(0, 2, 3, 4, 1)
        dist = m.quantizer.codebooks[0].compute_distances(z_pre)
        top2 = dist.topk(2, dim=-1, largest=False).values
        assert torch.equal(dist.argmin(-1), code.view(b, t, h, w))
        out_code = m.decode_code(code.view(Fr, h, w, 1))
        soft, soft_code = m.get_soft_codes(x.view(Fr, 3, H, W), temp=1.0)
    rec = {'seed': seed, 'b': b, 't': t, 'H': H, 'quant_loss': loss, 'codes': code.to(torch.int16),
           'margin': (top2[..., 1] - top2[..., 0]).contiguous(), 'soft_codes': soft_code.to(torch.int16)}
    tensors = {'z_e': (z_e, 'z'), 'z_pre': (z_pre.contiguous(), 'z'), 'z_q': (z_q.contiguous(), 'z'),
               'out': (out, 'out'), 'out_code': (out_code, 'out'), 'soft': (soft, 'soft')}
    if W != H:
        rec['W'] = W
    for key, (v, kind) in tensors.items():
        if strides is None:
            rec[key] = v.contiguous()
        else:
            sample_into(rec, key, v, strides[kind])
    if H >= 512:                                             # the compact fixture keeps its frame samples as fp16
        for key in ('out', 'out_code'):
            rec[key] = rec[key].to(torch.float16)
    path = os.path.join(GOLDEN, golden_name(seed, b, t, H, W if W != H else None))
    torch.save(rec, path)
    print('wrote %s in %.0f s (%.0f KB)' % (path, time.time() - t0, os.path.getsize(path) / 1e3))


def main():
    torch.set_num_threads(os.cpu_count())
    m = reference_model()
    write_spec(m)
    only = [int(a) for a in sys.argv[1:]]
    for (seed, b, t, H, *W), strides in CASES.items():
        if not only or H in only:
            mint(m, seed, b, t, H, strides, *W)


if __name__ == '__main__':
    main()
