"""The load-time weight pack (Engine._repack) of the six registered models, run on the CPU on their synthetic state
dicts: every state-dict tensor reaches a kernel layout, a fused transform, a prefix packed by a rule of its own or a
short list of entries no launch reads, and a packed conv or linear, unpacked, is its bf16-rounded source."""
import copy

import pytest
import torch

BF = torch.bfloat16
# entries no launch reads: the codebooks' EMA state (training only)
UNREAD = ('.embed_ema',)
# entries a fused transform consumes, with the key of what it becomes (relative to the entry's module)
FUSED = {'.relative_position_bias_table': '.bias_tab', '.relative_position_index': '.bias_tab',
         '.in_proj_weight': '.qk.weight'}

MODELS = ['PGTFormer', 'TDRQVAE', 'RQVAE_r1', 'RQVAE_r2', 'VQGAN', 'CodeFormer']


def packed(name, network_g):
    """(engine after _repack on the CPU, its state dict)."""
    from pgtformer_b200 import spec as S
    from pgtformer_b200.engine import Engine
    from pgtformer_b200.rqvae import RQVAEEngine
    from pgtformer_b200.tdrqvae import TDRQVAEEngine
    from pgtformer_b200.vqgan import CodeFormerEngine, VQGANEngine
    if name == 'PGTFormer':
        cls, (arch, spec) = Engine, S.build_spec(network_g)
    elif name == 'TDRQVAE':
        cls, (arch, spec) = TDRQVAEEngine, S.build_tdrqvae_spec(dict(network_g, type='TDRQVAE'))
    elif name.startswith('RQVAE'):
        from oracle.make_rqvae_golden import CONFIGS
        cls, (arch, spec) = RQVAEEngine, S.build_rqvae_spec(copy.deepcopy(CONFIGS[name[-2:]]))
    elif name == 'VQGAN':
        cls, (arch, spec) = VQGANEngine, S.build_vqgan_spec({})
    else:
        cls, (arch, spec) = CodeFormerEngine, S.build_codeformer_spec({})
    return repacked(cls, arch, spec)


def repacked(cls, arch, spec):
    """(engine of class cls after _repack of spec's synthetic state dict on the CPU, that state dict)."""
    from pgtformer_b200.weights import synth_state_dict
    eng = cls.__new__(cls)
    eng.arch, eng.dev, eng.w = arch, torch.device('cpu'), {}
    eng._sd = synth_state_dict(spec, 0)
    eng._repack()
    return eng, eng._sd


def unpack(name, t, p, arch):
    """The packed p of state-dict tensor t back in t's layout (bf16)."""
    if t.dim() == 1:
        return p
    co = t.shape[0]
    if name == arch.stem:                                  # [Cout, 3*k*k] with K index (ky*k + kx)*3 + c
        k = t.shape[2]
        return p[:, :3 * k * k].reshape(co, k, k, 3).permute(0, 3, 1, 2)
    if t.dim() == 4 and t.shape[2] == 3:                   # [Cout, 9 * CinPad] with K index tap * CinPad + c
        ci = t.shape[1]
        cp = p.shape[1] // 9
        assert not p.view(co, 9, cp)[:, :, ci:].any()
        return p.view(co, 9, cp)[:, :, :ci].reshape(co, 3, 3, ci).permute(0, 3, 1, 2)
    k = t[0].numel()                                       # [N, roundup(K, 8)]
    assert not p[:, k:].any()
    return p[:, :k].reshape(t.shape)


@pytest.mark.parametrize('model', MODELS)
def test_every_state_dict_entry_is_packed_or_accounted_for(model, network_g):
    eng, sd = packed(model, network_g)
    a, w = eng.arch, eng.w
    unmatched = []
    for name, t in sd.items():
        if name.startswith(a.packed_apart) or name.endswith(UNREAD) or name in a.codebooks:
            continue
        fused = [s for s in FUSED if name.endswith(s)]
        if fused:
            assert name[:-len(fused[0])] + FUSED[fused[0]] in w, name
            continue
        if name not in w:
            unmatched.append(name)
            continue
        if name in a.upsample_convs:                       # 2x2 phase weights; phases (0,0) / (1,1), taps (0,0) / (1,1)
            co, ci = t.shape[:2]                           # are the single 3x3 taps (0,0) / (2,2)
            p = w[name].view(4, co, 4, -1)
            assert torch.equal(p[0, :, 0, :ci], t[:, :, 0, 0].to(BF)), name
            assert torch.equal(p[3, :, 3, :ci], t[:, :, 2, 2].to(BF)), name
            continue
        want = t.float() if t.dim() == 1 else t.to(BF)
        assert torch.equal(unpack(name, t, w[name], a), want), name
    assert not unmatched, 'state-dict entries no packing rule matched: %s' % unmatched[:10]


@pytest.mark.parametrize('model', MODELS)
def test_fused_projections_and_codebooks(model, network_g):
    eng, sd = packed(model, network_g)
    a, w = eng.arch, eng.w
    for name in sd:
        if name.startswith(a.packed_apart):
            continue
        if name.endswith('.attn.kv.weight'):              # Swin: [q | kv]
            p = name[:-len('.kv.weight')]
            assert torch.equal(w[p + '.qkv.weight'], torch.cat([sd[p + '.q.weight'], sd[name]]).to(BF))
        if name.endswith('.proj_out.weight'):             # AttnBlock: [q | k | v]
            p = name[:-len('.proj_out.weight')]
            want = torch.cat([sd[p + '.%s.weight' % n] for n in 'qkv']).flatten(1).to(BF)
            assert torch.equal(w[p + '.qkv.weight'], want)
        if name.endswith('.in_proj_weight'):              # MHA: (q, k) and v
            p, E = name[:-len('.in_proj_weight')], sd[name].shape[1]
            assert torch.equal(w[p + '.qk.weight'], sd[name][:2 * E].to(BF))
            assert torch.equal(w[p + '.v.weight'], sd[name][2 * E:].to(BF))
    assert torch.equal(w['codebook'], sd[a.codebooks[0]])
    if eng.depth > 1:
        distinct = a.codebooks[:1 if a.shared_codebook else eng.depth]
        assert w['codebooks'].shape[0] == len(distinct)
        for d, k in enumerate(distinct):
            rows = sd[k].shape[0]
            assert torch.equal(w['codebooks'][d, :rows], sd[k]) and not w['codebooks'][d, rows:].any()
    # the prefixes packed by a rule of their own: BiSeNet's folded convs, the Video-Swin layers
    assert ('bn.stem.weight' in w) == ('conditionnet.' in a.packed_apart)
    assert sorted(eng.swin) == sorted(p[:-1] for p in a.packed_apart if p != 'conditionnet.')
