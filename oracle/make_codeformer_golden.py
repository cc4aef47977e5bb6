"""TEST INFRASTRUCTURE ONLY — mints tests/golden/vqgan_*.pt, tests/golden/codeformer_*.pt and their state-dict spec JSONs
from the UNMODIFIED reference's `archs/vqgan_arch.py` / `archs/codeformer_arch.py` (imported with the basicsr shim of
oracle/shims), built with default arguments and loaded with the deterministic synthetic checkpoint
(pgtformer_b200.weights.synth_state_dict of build_vqgan_spec / build_codeformer_spec, seed 0) with strict=True:

    PGT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_codeformer_golden

Inputs are in [-1, 1], as CodeFormer's users feed it, and are not stored: `golden_images(seed, b, H, W)` regenerates
them bit-exactly.  Fixtures (all compact; large tensors as strided flat samples, see make_golden.sample_into):
  VQAutoEncoder, b = 1, 512^2 and b = 2, 256 x 384: every code with its top-2 distance margin, the loss and the
    statistics, `usage` after the call, the encoder output z, out (fp16);
  CodeFormer, b = 1, 512^2: every code with its top-2 logit margin, some full logit rows, lq_feat, and out (fp16) for
    (w, adain) = (0, False), (0.5, True), (1, False); code_only is checked against the full forward while minting;
  CodeFormer, b = 2, 512^2, (0.5, True)."""
import contextlib
import io
import json
import os
import sys
import time

import torch

from oracle.make_golden import GOLDEN, sample_into

VQ_CASES = {(51, 1, 512, 512): {'z': 4, 'out': 16}, (52, 2, 256, 384): {'z': 4, 'out': 16}}
CF_CASES = {(61, 1): ((0.0, False), (0.5, True), (1.0, False)), (62, 2): ((0.5, True),)}
CF_STRIDES = {'lq_feat': 4, 'out': 16}
N_LOGIT_ROWS = 16


def golden_images(seed, b, H, W):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 3, H, W, generator=g) * 2 - 1


def vq_name(seed, b, H, W):
    return 'vqgan_ref_b%d_%dx%d_seed%d.pt' % (b, H, W, seed)


def cf_name(seed, b):
    return 'codeformer_ref_b%d_512_seed%d.pt' % (b, seed)


def logit_rows(T, seed):
    g = torch.Generator().manual_seed(2000 + seed)
    return torch.randperm(T, generator=g)[:N_LOGIT_ROWS].sort().values


def import_reference_codeformer():
    """The reference's `archs.codeformer_arch` module (which imports its `archs.vqgan_arch`), imported from
    PGT_REFERENCE_ROOT with the repo's own `archs` package set aside while importing and restored afterwards."""
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
            import archs.codeformer_arch as ref_mod
        ref_pkg = {k: v for k, v in sys.modules.items() if own(k)}
    finally:
        os.chdir(cwd)
        sys.path = saved_path
    for k, v in ref_pkg.items():
        sys.modules['_pgt_reference_codeformer.' + k] = v
        del sys.modules[k]
    sys.modules.update(saved)
    return ref_mod


def reference_models():
    from pgtformer_b200.spec import build_codeformer_spec, build_vqgan_spec
    from pgtformer_b200.weights import synth_state_dict
    ref = import_reference_codeformer()
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        vq, cf = ref.VQAutoEncoder(), ref.CodeFormer()
    vq.load_state_dict(synth_state_dict(build_vqgan_spec({})[1], 0), strict=True)
    cf.load_state_dict(synth_state_dict(build_codeformer_spec({})[1], 0), strict=True)
    for m in (vq, cf):
        m.eval()
        for p in m.parameters():
            p.requires_grad_(False)
    return vq, cf


def write_spec(m, name):
    spec = {k: [list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()}
    path = os.path.join(GOLDEN, name)
    with open(path, 'w') as f:
        json.dump(spec, f, indent=0, sort_keys=False)
        f.write('\n')
    print('wrote %s (%d entries)' % (path, len(spec)))


def _save(rec, name, t0):
    path = os.path.join(GOLDEN, name)
    torch.save(rec, path)
    print('wrote %s in %.0f s (%.0f KB)' % (path, time.time() - t0, os.path.getsize(path) / 1e3))


def mint_vq(m, seed, b, H, W, strides):
    t0 = time.time()
    x = golden_images(seed, b, H, W)
    m.quantize.reset_usage()
    with torch.no_grad():
        z = m.encoder(x)
        out, loss, st = m(x)
        usage = m.quantize.usage.clone()
        quant, loss2, st2 = m(x, code_only=True)
        zf = z.permute(0, 2, 3, 1).reshape(-1, z.shape[1])
        emb = m.quantize.embedding.weight
        d = (zf ** 2).sum(1, keepdim=True) + (emb ** 2).sum(1) - 2 * zf @ emb.t()
        top2 = d.topk(2, dim=1, largest=False).values
    assert torch.equal(st['min_encoding_indices'], st2['min_encoding_indices']) and torch.equal(loss, loss2)
    rec = {'seed': seed, 'b': b, 'H': H, 'W': W, 'codes': st['min_encoding_indices'].view(-1).to(torch.int16),
           'margin': (top2[:, 1] - top2[:, 0]).contiguous(), 'loss': loss, 'perplexity': st['perplexity'],
           'mean_distance': st['mean_distance'], 'scores': st['min_encoding_scores'].view(-1).contiguous(),
           'usage': usage.to(torch.int16)}
    sample_into(rec, 'z', z, strides['z'])
    sample_into(rec, 'quant', quant, strides['z'])
    sample_into(rec, 'out', out, strides['out'])
    rec['out'] = rec['out'].to(torch.float16)
    _save(rec, vq_name(seed, b, H, W), t0)


def mint_cf(m, seed, b, cases):
    t0 = time.time()
    x = golden_images(seed, b, 512, 512)
    with torch.no_grad():
        logits, lq = m(x, code_only=True)
        outs = {}
        for w, adain in cases:
            out, logits2, lq2 = m(x, w=w, adain=adain)
            assert torch.equal(logits, logits2) and torch.equal(lq, lq2)
            outs[(w, adain)] = out
    T = logits.shape[0] * logits.shape[1]
    lg = logits.reshape(T, -1)
    top2 = lg.topk(2, dim=1).values
    rows = logit_rows(T, seed)
    codes = torch.topk(torch.softmax(logits, dim=2), 1, dim=2)[1].reshape(-1)
    rec = {'seed': seed, 'b': b, 'cases': list(cases), 'codes': codes.to(torch.int16),
           'margin': (top2[:, 0] - top2[:, 1]).contiguous(), 'logit_rows': rows, 'logits_sel': lg[rows].contiguous(),
           'logits_shape': tuple(logits.shape), 'logits_absmax': logits.abs().max().item()}
    sample_into(rec, 'lq_feat', lq, CF_STRIDES['lq_feat'] * b)
    for i, key in enumerate(cases):
        sample_into(rec, 'out%d' % i, outs[key], CF_STRIDES['out'] * b)
        rec['out%d' % i] = rec['out%d' % i].to(torch.float16)
    _save(rec, cf_name(seed, b), t0)


def main():
    torch.set_num_threads(os.cpu_count())
    vq, cf = reference_models()
    write_spec(vq, 'vqgan_state_dict_spec.json')
    write_spec(cf, 'codeformer_state_dict_spec.json')
    for (seed, b, H, W), strides in VQ_CASES.items():
        mint_vq(vq, seed, b, H, W, strides)
    for (seed, b), cases in CF_CASES.items():
        mint_cf(cf, seed, b, cases)


if __name__ == '__main__':
    main()
