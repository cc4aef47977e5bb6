"""TEST INFRASTRUCTURE ONLY — mints tests/golden/tdcrqvae3_codec_*.pt from the UNMODIFIED reference's TDCRQVAE3
methods (`archs/tdcrqvae3_arch.py:774-813`, RQBottleneck.get_soft_codes :429-457), called unbound on the reference
module with the deterministic synthetic checkpoint (seed 0) and the size patch, one clip at a time (SURVEY F5):

    PGT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_codec_golden

64^2, b = 1 (kept whole): encode, decode of the quantiser's z_q, decode_code of a seeded code map that includes the
padding row, and get_soft_codes at three temperatures (in a file of their own, so each file stays below 1 MB).
128^2, b = 2 and 64x192, b = 1: strided samples of encode and of decode of the codebook rows of the reference's own
codes; at 64x192 also decode_code of a seeded code map.
Inputs are not stored: `oracle.make_golden.golden_input(seed, b, H, W)` regenerates them bit-exactly."""
import os

import torch
import torch.nn.functional as F

from oracle.make_golden import GOLDEN, _reference_model, golden_input, sample_into

CODEC_TEMPS = (1.0, 10.0, 100.0)
CODEC_STRIDES = {'z_e': 4, 'out': 4}                # 128^2, b = 2 and 64x192


def codec_code_map(seed, Fr, h, w, n_embed):
    """Seeded code map [Fr, h, w, 1] over [0, n_embed], the padding row n_embed included."""
    g = torch.Generator().manual_seed(seed)
    code = torch.randint(0, n_embed + 1, (Fr, h, w, 1), generator=g)
    code.view(-1)[::7] = n_embed
    return code


def main():
    from oracle.reference_loader import generalise_size, import_reference
    ref_mod = import_reference()
    m = _reference_model()
    V = ref_mod.TDCRQVAE3
    n_embed = m.quantizer.n_embed[0]
    seed, H = 21, 64
    generalise_size(m, H, H)
    x = golden_input(seed, 1, H)
    xs = x.view(1, 3, 3, H, H)
    with torch.no_grad():
        z_e = V.encode(m, xs)
        z_q, _, codes = m.quantizer(z_e)
        out = V.decode(m, z_q)
        code = codec_code_map(seed, 3, H // 16, H // 16, n_embed)
        out_code = V.decode_code(m, code)
        soft = [V.get_soft_codes(m, xs, temp=t) for t in CODEC_TEMPS]
    rec = {'seed': seed, 'b': 1, 'H': H, 'z_e': z_e, 'z_q': z_q, 'codes': codes, 'out': out, 'code': code,
           'out_code': out_code}
    path = os.path.join(GOLDEN, 'tdcrqvae3_codec_b1_%d_seed%d.pt' % (H, seed))
    torch.save(rec, path)
    print('wrote %s (%.0f KB)' % (path, os.path.getsize(path) / 1e3))
    rec = {'seed': seed, 'b': 1, 'H': H, 'temps': CODEC_TEMPS, 'soft_code': [s[0] for s in soft],
           'code': [s[1] for s in soft]}
    path = os.path.join(GOLDEN, 'tdcrqvae3_codec_soft_b1_%d_seed%d.pt' % (H, seed))
    torch.save(rec, path)
    print('wrote %s (%.0f KB)' % (path, os.path.getsize(path) / 1e3))
    # 128^2, two clips; decode input = the codebook rows of the reference's own codes
    seed, b, H = 22, 2, 128
    x = golden_input(seed, b, H)
    zs, outs, cs = [], [], []
    with torch.no_grad():
        for i in range(b):
            generalise_size(m, H, H)
            z = V.encode(m, x[i * 3:(i + 1) * 3].view(1, 3, 3, H, H))
            c = m.quantizer(z)[2]
            zs.append(z)
            cs.append(c)
            outs.append(V.decode(m, F.embedding(c[..., 0], m.quantizer.codebooks[0].weight)))
    rec = {'seed': seed, 'b': b, 'H': H, 'codes': torch.cat(cs, 0)}
    sample_into(rec, 'z_e', torch.cat(zs, 0), CODEC_STRIDES['z_e'])
    sample_into(rec, 'out', torch.cat(outs, 0), CODEC_STRIDES['out'])
    path = os.path.join(GOLDEN, 'tdcrqvae3_codec_b%d_%d_seed%d.pt' % (b, H, seed))
    torch.save(rec, path)
    print('wrote %s (%.0f KB)' % (path, os.path.getsize(path) / 1e3))
    # 64x192: level 4 and the mid layers are one window row deep, where only x is shifted (get_window_size per axis)
    seed, H, W = 23, 64, 192
    generalise_size(m, H, W)
    x = golden_input(seed, 1, H, W)
    with torch.no_grad():
        z_e = V.encode(m, x.view(1, 3, 3, H, W))
        codes = m.quantizer(z_e)[2]
        out = V.decode(m, F.embedding(codes[..., 0], m.quantizer.codebooks[0].weight))
        code = codec_code_map(seed, 3, H // 16, W // 16, n_embed)
        out_code = V.decode_code(m, code)
    rec = {'seed': seed, 'b': 1, 'H': H, 'W': W, 'codes': codes, 'code': code}
    sample_into(rec, 'z_e', z_e, CODEC_STRIDES['z_e'])
    sample_into(rec, 'out', out, CODEC_STRIDES['out'])
    sample_into(rec, 'out_code', out_code, CODEC_STRIDES['out'])
    path = os.path.join(GOLDEN, 'tdcrqvae3_codec_b1_%dx%d_seed%d.pt' % (H, W, seed))
    torch.save(rec, path)
    print('wrote %s (%.0f KB)' % (path, os.path.getsize(path) / 1e3))


if __name__ == '__main__':
    main()
