"""TEST INFRASTRUCTURE ONLY — mints tests/golden/rq_*.pt / rq_state_dict_specs.json from the UNMODIFIED reference's
residual quantiser at depth D > 1 (RQBottleneck, `archs/tdcrqvae3_arch.py:206-457`; TDCRQVAE3's methods :760-872;
PGTFormer.forward `archs/pgtformer_arch.py:598-714`), with the deterministic synthetic checkpoint (seed 0) of each
configuration and the size patch, one clip at a time:

    PGT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_rq_golden

Configurations: TDCRQVAE3 at D = 2 with separate codebooks and D = 4 with one shared codebook; PGTFormer at D = 2
(shared, as in the options files).  The size patch (`reference_loader.generalise_size`) sets code_shape to
[H/16, W/16, 1]; the depth is put back after it.  Inputs are not stored: `make_golden.golden_input` and `rq_inputs`
regenerate them bit-exactly.  Every file stays below 1 MB (large tensors as strided samples, `make_golden.sample_into`).
"""
import json
import os

import torch

from oracle.make_golden import GOLDEN, golden_input, load_network_g, sample_into

CONFIGS = {'d2_separate': (2, False), 'd4_shared': (4, True)}      # TDCRQVAE3: name -> (depth, shared_codebook)
PGT_DEPTH = 2
SOFT_TEMPS = (1.0, 30.0)
RQ_ALONE = dict(T=4096, K=1024, E=512, D=4, seed=41)


def network_g(depth, shared):
    g = load_network_g()
    g['code_shape'] = [32, 32, depth]
    g['shared_codebook'] = shared
    return g


def rq_inputs(T, K, E, D, seed):
    """Seeded z [T, E] and D codebook weights [K + 1, E] (padding row zero) for the RQBottleneck-alone case: depth d's
    codebook is scaled by 0.5^d, so each level quantises what the coarser ones left."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(T, E, generator=g)
    cbs = []
    for d in range(D):
        w = torch.randn(K + 1, E, generator=g) * 0.5 ** d
        w[-1].zero_()
        cbs.append(w)
    return z, cbs


def code_map(seed, Fr, h, w, D, n_embed):
    """Seeded codes [Fr, h, w, D] over [0, n_embed], the padding row included."""
    g = torch.Generator().manual_seed(seed)
    code = torch.randint(0, n_embed + 1, (Fr, h, w, D), generator=g)
    code.view(-1)[::7] = n_embed
    return code


def _model(g):
    from oracle.reference_loader import build_reference_model
    from pgtformer_b200.spec import build_spec
    from pgtformer_b200.weights import synth_state_dict
    _, spec = build_spec(g)
    torch.set_num_threads(os.cpu_count())
    return build_reference_model(g, synth_state_dict(spec, 0))


def _size(m, H, D):
    from oracle.reference_loader import generalise_size
    generalise_size(m, H, H)
    m.quantizer.code_shape = torch.Size([H // 16, H // 16, D])


def _save(rec, name):
    path = os.path.join(GOLDEN, name)
    torch.save(rec, path)
    print('wrote %s (%.0f KB)' % (path, os.path.getsize(path) / 1e3))
    assert os.path.getsize(path) < 1e6, path


def state_dict_spec(m):
    """Names, shapes, dtypes and alias groups (keys sharing one tensor) of a reference module's state dict."""
    sd = m.state_dict()
    groups = {}
    for k, v in sd.items():
        groups.setdefault(v.data_ptr(), []).append(k)
    return {'keys': [[k, list(v.shape), str(v.dtype).replace('torch.', '')] for k, v in sd.items()],
            'aliases': [g for g in groups.values() if len(g) > 1]}


def rq_alone():
    from oracle.reference_loader import import_reference
    ref = import_reference()
    RQ = ref.TDCRQVAE3.__init__.__globals__['RQBottleneck']            # the class of archs/tdcrqvae3_arch.py:206
    c = RQ_ALONE
    z, cbs = rq_inputs(**c)
    q = RQ(latent_shape=[64, 64, c['E']], code_shape=[64, 64, c['D']], n_embed=c['K'], shared_codebook=False)
    q.eval()
    with torch.no_grad():
        for d in range(c['D']):
            q.codebooks[d].weight.copy_(cbs[d])
        quant_list, codes = q.quantize(z.view(1, 64, 64, c['E']))
    rec = dict(c, codes=codes.view(c['T'], c['D']))
    for d, ql in enumerate(quant_list):
        sample_into(rec, 'quant_%d' % d, ql.view(c['T'], c['E']), 61)
    _save(rec, 'rq_bottleneck_T%d_K%d_E%d_D%d_seed%d.pt' % (c['T'], c['K'], c['E'], c['D'], c['seed']))


def codec(name, depth, shared):
    from oracle.reference_loader import import_reference
    V = import_reference().TDCRQVAE3
    m = _model(network_g(depth, shared))
    n_embed = m.quantizer.n_embed[0]
    seed, H = 51 + depth, 64
    _size(m, H, depth)
    x = golden_input(seed, 1, H)
    xs = x.view(1, 3, 3, H, H)
    with torch.no_grad():
        z_e = V.encode(m, xs)
        z_q, loss, codes = m.quantizer(z_e)
        out = V.decode(m, z_q)
        code = code_map(seed, 3, H // 16, H // 16, depth, n_embed)
        out_code = V.decode_code(m, code)
        emb, _ = V.get_code_emb_with_depth(m, code)
        partial = {(j, t): V.decode_partial_code(m, code, j, t) for j in range(depth) for t in ('select', 'add')}
        soft = [V.get_soft_codes(m, xs, temp=t) for t in SOFT_TEMPS]
    rec = {'seed': seed, 'b': 1, 'H': H, 'depth': depth, 'shared': shared, 'z_e': z_e, 'z_q': z_q, 'loss': loss,
           'codes': codes, 'code': code, 'temps': SOFT_TEMPS, 'soft_code_codes': [s[1] for s in soft]}
    sample_into(rec, 'emb_with_depth', emb, 3)
    sample_into(rec, 'out', out, 3)
    sample_into(rec, 'out_code', out_code, 3)
    for (j, t), o in partial.items():
        sample_into(rec, 'partial_%s_%d' % (t, j), o, 7)
    for i, s in enumerate(soft):
        sample_into(rec, 'soft_code_%d' % i, s[0], 7)
    _save(rec, 'rq_tdcrqvae3_%s_b1_%d_seed%d.pt' % (name, H, seed))
    # 128^2, two clips, one at a time
    seed, b, H = 61 + depth, 2, 128
    x = golden_input(seed, b, H)
    zs, zqs, cs, outs = [], [], [], []
    with torch.no_grad():
        for i in range(b):
            _size(m, H, depth)
            z = V.encode(m, x[i * 3:(i + 1) * 3].view(1, 3, 3, H, H))
            zq, _, c = m.quantizer(z)
            zs.append(z)
            zqs.append(zq)
            cs.append(c)
            outs.append(V.decode(m, zq))
    rec = {'seed': seed, 'b': b, 'H': H, 'depth': depth, 'shared': shared, 'codes': torch.cat(cs, 0)}
    sample_into(rec, 'z_e', torch.cat(zs, 0), 5)
    sample_into(rec, 'z_q', torch.cat(zqs, 0), 5)
    sample_into(rec, 'out', torch.cat(outs, 0), 5)
    _save(rec, 'rq_tdcrqvae3_%s_b%d_%d_seed%d.pt' % (name, b, H, seed))


def pgtformer():
    m = _model(network_g(PGT_DEPTH, True))
    for seed, b, H in ((71, 1, 64), (72, 2, 128)):
        x = golden_input(seed, b, H)
        outs = []
        with torch.no_grad():
            for i in range(b):
                _size(m, H, PGT_DEPTH)
                outs.append(m(x[i * 3:(i + 1) * 3], w=1.0, adain=True))
        out, logits, lq = (torch.cat([o[j] for o in outs], 0) for j in range(3))
        rec = {'seed': seed, 'b': b, 'H': H, 'depth': PGT_DEPTH, 'w': 1.0, 'adain': True, 'codes': logits.argmax(-1),
               'top2': logits.topk(2, dim=-1).values}
        sample_into(rec, 'out', out, 2 * b)
        sample_into(rec, 'lq_feat', lq.contiguous(), 2 * b)
        sample_into(rec, 'logits', logits, 5 * b)
        _save(rec, 'rq_pgtformer_d%d_b%d_%d_seed%d.pt' % (PGT_DEPTH, b, H, seed))


def main(parts):
    """parts: any of 'alone', the CONFIGS names, 'pgtformer', 'specs' (default: all)."""
    if 'alone' in parts:
        rq_alone()
    for name, (depth, shared) in CONFIGS.items():
        if name in parts:
            codec(name, depth, shared)
    if 'pgtformer' in parts:
        pgtformer()
    if 'specs' not in parts:
        return
    specs = {'pgtformer_' + name: state_dict_spec(_model(network_g(depth, shared)))
             for name, (depth, shared) in CONFIGS.items()}
    specs['pgtformer_d%d_shared' % PGT_DEPTH] = state_dict_spec(_model(network_g(PGT_DEPTH, True)))
    path = os.path.join(GOLDEN, 'rq_state_dict_specs.json')
    with open(path, 'w') as f:
        json.dump(specs, f)
    print('wrote', path, '(%.0f KB)' % (os.path.getsize(path) / 1e3))


if __name__ == '__main__':
    import sys
    main(sys.argv[1:] or ['alone', *CONFIGS, 'pgtformer', 'specs'])
