"""TEST INFRASTRUCTURE ONLY — mints tests/golden/rqvae_*.pt and tests/golden/rqvae_{r1,r2}_state_dict_spec.json from the
UNMODIFIED reference's `archs/rqvae_arch.py` (imported with the basicsr shim of oracle/shims), built from the two
configurations below and loaded with the deterministic synthetic checkpoint (pgtformer_b200.weights.synth_state_dict of
build_rqvae_spec, seed 0) with strict=True:

    PGT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_rqvae_golden

R1 is the f = 32 shape of Kakao Brain's released 8x8x4 RQ-VAEs (ch 128, six levels, attention at 8^2, a shared codebook
of 2048 codes); R2 a 64-wide f = 8 model with separate codebooks of different sizes.  The reference's get_soft_codes
concatenates the depths' soft codes, which fails for codebooks of different sizes, so R2 has no soft-code sample.

Fixtures (inputs are not stored: `golden_images(seed, b, H, W)` regenerates them bit-exactly) record z_e = encode(x),
every code with the top-2 distance margin of its depth's residual, quant_loss, the code_only z_q, out, decode_code of the
reference's own codes, decode_partial_code ('select' and 'add' at depth 1) and, for R1, a soft-code sample (temp 1).
Large tensors are strided flat samples.  Away from the configured resolution the decode methods need the
`quantizer.code_shape` patch applied in mint()."""
import contextlib
import io
import json
import os
import sys
import time

import torch

from oracle.make_golden import GOLDEN, sample_into

R1 = {'type': 'RQVAE', 'embed_dim': 256, 'n_embed': 2048, 'decay': 0.99, 'loss_type': 'mse', 'latent_loss_weight': 0.25,
      'bottleneck_type': 'rq', 'latent_shape': [8, 8, 256], 'code_shape': [8, 8, 4], 'shared_codebook': True,
      'restart_unused_codes': True,
      'ddconfig': {'double_z': False, 'z_channels': 256, 'resolution': 256, 'in_channels': 3, 'out_ch': 3, 'ch': 128,
                   'ch_mult': [1, 1, 2, 2, 4, 4], 'num_res_blocks': 2, 'attn_resolutions': [8], 'dropout': 0.0}}
R2 = {'type': 'RQVAE', 'embed_dim': 128, 'n_embed': [512, 1024, 256], 'decay': 0.99, 'loss_type': 'mse',
      'latent_loss_weight': 0.25, 'bottleneck_type': 'rq', 'latent_shape': [16, 16, 128], 'code_shape': [16, 16, 3],
      'shared_codebook': False, 'restart_unused_codes': True,
      'ddconfig': {'double_z': False, 'z_channels': 256, 'resolution': 128, 'in_channels': 3, 'out_ch': 3, 'ch': 64,
                   'ch_mult': [1, 2, 2, 4], 'num_res_blocks': 2, 'attn_resolutions': [16], 'dropout': 0.0}}
CONFIGS = {'r1': R1, 'r2': R2}
# (config, seed, b, H, W) -> flat sample strides of the large tensors; latents are kept whole (per-token code checks)
CASES = {('r1', 81, 1, 256, 256): {'z': 1, 'out': 16, 'soft': 64},
         ('r1', 82, 2, 256, 256): {'z': 1, 'out': 32, 'soft': 128},
         ('r2', 83, 2, 128, 128): {'z': 1, 'out': 16},
         ('r2', 84, 1, 128, 256): {'z': 1, 'out': 16}}


def spec_json(cfg):
    return os.path.join(GOLDEN, 'rqvae_%s_state_dict_spec.json' % cfg)


def golden_images(seed, b, H, W):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 3, H, W, generator=g)


def golden_name(cfg, seed, b, H, W):
    return 'rqvae_%s_b%d_%dx%d_seed%d.pt' % (cfg, b, H, W, seed)


def import_reference_rqvae():
    """The reference's `archs.rqvae_arch` module, imported from PGT_REFERENCE_ROOT with the names `archs` / `modules`
    resolving to the reference's while importing; the repo's own packages are restored afterwards."""
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
        os.chdir(REFERENCE_ROOT)
        with contextlib.redirect_stdout(io.StringIO()):
            import archs.rqvae_arch as ref_mod
        ref_pkg = {k: v for k, v in sys.modules.items() if own(k)}
    finally:
        os.chdir(cwd)
        sys.path = saved_path
    for k, v in ref_pkg.items():
        sys.modules['_pgt_reference_rqvae.' + k] = v
        del sys.modules[k]
    sys.modules.update(saved)
    return ref_mod


def reference_model(ref_mod, g):
    from pgtformer_b200.spec import build_rqvae_spec
    from pgtformer_b200.weights import synth_state_dict
    _, spec = build_rqvae_spec(g)
    opt = dict(g)
    opt.pop('type')
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):          # the reference's Decoder prints its z shape
        m = ref_mod.RQVAE(**opt)
    m.eval()
    m.load_state_dict(synth_state_dict(spec, 0), strict=True)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def write_spec(m, cfg):
    spec = {k: [list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()}
    with open(spec_json(cfg), 'w') as f:
        json.dump(spec, f, indent=0, sort_keys=False)
        f.write('\n')
    print('wrote %s (%d entries)' % (spec_json(cfg), len(spec)))


def mint(m, cfg, seed, b, H, W, strides):
    x = golden_images(seed, b, H, W)
    t0 = time.time()
    q = m.quantizer
    with torch.no_grad():
        out, loss, code = m(x)
        z_q, loss2, code2 = m(x, code_only=True)
        assert torch.equal(code, code2) and torch.equal(loss, loss2)
        z_e = m.encode(x)
        # embed_code / embed_partial_code assert the constructor's code_shape; decoding codes of another image size
        # needs it patched to the codes' shape (as reference_loader.generalise_size does for the other models)
        q.code_shape = torch.Size(code.shape[1:])
        # each depth's top-2 distance margin on the residual the earlier depths left (RQBottleneck.quantize, :436-440)
        r, margins = z_e.clone(), []
        for d in range(code.shape[-1]):
            dist = q.codebooks[d].compute_distances(r)
            top2 = dist.topk(2, dim=-1, largest=False).values
            assert torch.equal(dist.argmin(-1), code[..., d])
            margins.append(top2[..., 1] - top2[..., 0])
            r -= q.codebooks[d].embed(code[..., d])
        out_code = m.decode_code(code)
        sel = m.decode_partial_code(code, 1, 'select')
        add = m.decode_partial_code(code, 1, 'add')
        soft = None
        if len(set(q.n_embed)) == 1:
            soft, soft_code = m.get_soft_codes(x, temp=1.0)
    rec = {'config': cfg, 'seed': seed, 'b': b, 'H': H, 'W': W, 'quant_loss': loss, 'codes': code.to(torch.int16),
           'margin': torch.stack(margins, -1).contiguous()}
    tensors = {'z_e': (z_e, 'z'), 'z_q': (z_q.contiguous(), 'z'), 'out': (out, 'out'), 'out_code': (out_code, 'out'),
               'out_select1': (sel, 'out'), 'out_add1': (add, 'out')}
    if soft is not None:
        rec['soft_codes'] = soft_code.to(torch.int16)
        tensors['soft'] = (soft.contiguous(), 'soft')
    for key, (v, kind) in tensors.items():
        sample_into(rec, key, v, strides[kind])
    path = os.path.join(GOLDEN, golden_name(cfg, seed, b, H, W))
    torch.save(rec, path)
    print('wrote %s in %.0f s (%.0f KB)' % (path, time.time() - t0, os.path.getsize(path) / 1e3))


def main():
    torch.set_num_threads(os.cpu_count())
    ref_mod = import_reference_rqvae()
    for cfg, g in CONFIGS.items():
        m = reference_model(ref_mod, g)
        write_spec(m, cfg)
        for (c, seed, b, H, W), strides in CASES.items():
            if c == cfg:
                mint(m, cfg, seed, b, H, W, strides)


if __name__ == '__main__':
    main()
