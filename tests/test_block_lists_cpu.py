"""The block lists the engines walk and the state-dict layouts the spec builders write agree beyond the configurations
of the reference fixtures: over a grid of configurations of the six registered models, run on the CPU with every kernel
call replaced by test_walk_cpu's recorder, every `encoder.` / `decoder.` / `generator.` block the spec declares is read
by some call, and no call looks up a weight the spec does not declare."""
import copy
import re

import pytest
import torch

from test_pack_cpu import repacked
from test_walk_cpu import _calls, install

# the block a weight belongs to: one ResBlock, AttnBlock, Swin layer, resampling conv, norm or conv of the walk
BLOCK = re.compile(r'(?:encoder|decoder|generator)\.(?:blocks\.\d+|(?:down|up)\.\d+\.(?:block|attn)\.\d+|'
                   r'(?:down|up)\.\d+\.(?:downsample|upsample)|mid\.\w+?(?=\.)|\w+?(?=\.))')


def _levels(*ch_mult):
    n = len(ch_mult)
    return {'ch_mult': list(ch_mult), 'depths': [2] * n, 'num_heads': [8] * n, 'window_sizes': [[4, 4]] * n}


def _rq(depth, shared, side):
    return {'code_shape': [side, side, depth], 'shared_codebook': shared}


# (model, id, top-level overrides (None: the key left out), ddconfig overrides), TDCRQVAE3 / PGTFormer / TDRQVAE on the
# options file's network_g, RQVAE on the R2 fixture configuration, VQGAN and CodeFormer on their constructor defaults
GRID = [('TDCRQVAE3', 'r%d' % r, {}, {'num_res_blocks': r}) for r in (1, 2, 3)] + \
    [('TDCRQVAE3', 'attn%d' % len(a), {}, {'attn_resolutions': a}) for a in ([], [32], [32, 64])] + \
    [('TDCRQVAE3', 'levels%d' % len(m), {}, _levels(*m)) for m in ((1, 2, 4), (1, 2, 4, 8), (1, 1, 2, 4, 4, 8))] + \
    [('TDCRQVAE3', 'd%d_%s' % (d, 'shared' if s else 'separate'), _rq(d, s, 32), {})
     for d in (1, 2, 4) for s in (True, False)] + \
    [('TDCRQVAE3', 'd2_shared_default', _rq(2, None, 32), {})] + \
    [('PGTFormer', 'r2', {}, {'num_res_blocks': 2}), ('PGTFormer', 'attn1', {}, {'attn_resolutions': [32]}),
     ('PGTFormer', 'd2_separate', _rq(2, False, 32), {})] + \
    [('PGTFormer', 'connect_' + ('_'.join(c) or 'none'), {'connect_list': c}, {})
     for c in ([], ['32'], ['64', '256'])] + \
    [('TDRQVAE', 'r%d' % r, {}, {'num_res_blocks': r}) for r in (1, 2, 3)] + \
    [('TDRQVAE', 'attn%d' % len(a), {}, {'attn_resolutions': a}) for a in ([], [32], [32, 64])] + \
    [('TDRQVAE', 'levels%d' % len(m), {}, dict(_levels(*m), attn_resolutions=a))
     for m, a in (((1, 4, 8), [128]), ((1, 2, 4, 8), [32, 64, 128]), ((1, 1, 2, 4, 4, 8), [32]))] + \
    [('RQVAE', 'd%d_%s' % (d, 'shared' if s else 'separate'), dict(_rq(d, s, 16), n_embed=512), {})
     for d in (1, 2, 4) for s in (True, False)] + \
    [('RQVAE', 'd2_sizes', dict(_rq(2, False, 16), n_embed=[256, 512]), {})] + \
    [('RQVAE', 'r%d' % r, {}, {'num_res_blocks': r}) for r in (1, 3)] + \
    [('VQGAN', 'res_blocks%d' % r, {'res_blocks': r}, {}) for r in (1, 3)] + \
    [('VQGAN', 'levels4', {'ch_mult': [1, 2, 2, 4], 'attn_resolutions': [64]}, {})] + \
    [('CodeFormer', 'connect_' + ('_'.join(c) or 'none'), {'connect_list': c}, {})
     for c in ([], ['32'], ['16', '512'], ['64', '128', '256'], ['16', '32', '64', '128', '256', '512'])]

SIZES = {'TDCRQVAE3': (1, 128, 128), 'PGTFormer': (1, 64, 64), 'TDRQVAE': (1, 128, 128), 'RQVAE': (1, 128, 128),
         'VQGAN': (1, 128, 128), 'CodeFormer': (1, 512, 512)}


def config(model, top, dd, network_g):
    """The constructor keywords of one grid configuration of an RQ model."""
    if model == 'RQVAE':
        from oracle.make_rqvae_golden import CONFIGS
        g = copy.deepcopy(CONFIGS['r2'])
    else:
        g = dict(copy.deepcopy(network_g), type=model)
    g.update(top)
    g['ddconfig'].update(dd)
    return {k: v for k, v in g.items() if v is not None}


def build(model, top, dd, network_g):
    """(engine class, arch, spec) of one grid configuration."""
    from pgtformer_b200 import spec as S
    from pgtformer_b200.engine import Engine
    from pgtformer_b200.rqvae import RQVAEEngine
    from pgtformer_b200.tdrqvae import TDRQVAEEngine
    from pgtformer_b200.vqgan import CodeFormerEngine, VQGANEngine
    if model in ('VQGAN', 'CodeFormer'):
        return (CodeFormerEngine if model == 'CodeFormer' else VQGANEngine,
                *S.build_vqgan_spec(top, codeformer=model == 'CodeFormer'))
    g = config(model, top, dd, network_g)
    if model == 'TDRQVAE':
        return (TDRQVAEEngine, *S.build_tdrqvae_spec(g))
    if model == 'RQVAE':
        return (RQVAEEngine, *S.build_rqvae_spec(g))
    return (Engine, *S.build_spec(g))


class ReadLog(dict):
    """An engine's packed weights, recording every key its launches look up."""

    def __init__(self, w):
        super().__init__(w)
        self.read, self.missed = set(), set()

    def _log(self, k):
        (self.read if k in self else self.missed).add(k)

    def __getitem__(self, k):
        self._log(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        self._log(k)
        return super().get(k, default)


def _blocks(names):
    return {m.group(0) for m in map(BLOCK.match, names) if m}


@pytest.mark.parametrize('model,cid,top,dd', GRID, ids=['%s-%s' % (g[0], g[1]) for g in GRID])
def test_walk_reads_every_declared_block_and_nothing_else(network_g, monkeypatch, model, cid, top, dd):
    cls, arch, spec = build(model, top, dd, network_g)
    eng, _ = repacked(cls, arch, spec)
    install(monkeypatch)
    eng.w = log = ReadLog(eng.w)
    b, H, W = SIZES[model]
    for _, thunk in _calls(model, eng, b, H, W):
        thunk()
    declared = _blocks(spec)
    assert declared, 'no block matched'
    assert not {k for k in log.missed if k.startswith(('encoder.', 'decoder.', 'generator.'))}, sorted(log.missed)
    unread = declared - _blocks(log.read)
    assert not unread, 'declared blocks no call reads: %s' % sorted(unread)
    assert _blocks(log.read) <= declared


RQ_GRID = [g for g in GRID if g[0] in ('TDCRQVAE3', 'PGTFormer', 'TDRQVAE', 'RQVAE')]


@pytest.mark.parametrize('model,cid,top,dd', RQ_GRID, ids=['%s-%s' % (g[0], g[1]) for g in RQ_GRID])
def test_quantiser_description_agrees_with_the_state_dict_and_the_launches(network_g, monkeypatch, model, cid, top,
                                                                           dd):
    """The arch's depth, per-depth codebook sizes and codebook sharing are the model's `quantizer.` entries and aliases;
    every depth's embed_ema is its codebook without the padding row; and the engine's argmin of depth d scans that
    depth's K codes."""
    import archs  # noqa: F401
    from pgtformer_b200.registry import ARCH_REGISTRY
    cls = build(model, top, dd, network_g)[0]
    m = ARCH_REGISTRY.get(model)(**config(model, top, dd, network_g))
    a, spec, sd = m.arch, m._spec, m.state_dict()
    D = a.depth
    assert D == a.code_shape[2] == len(a.n_embeds) >= 1 and a.n_embed == max(a.n_embeds)
    quantizer = {k.rsplit('.', 1)[0] for k in spec if k.startswith('quantizer.')}
    assert quantizer == {'quantizer.codebooks.%d' % d for d in range(D)}
    for d, k in enumerate(a.n_embeds):
        p = 'quantizer.codebooks.%d.' % d
        assert spec[p + 'weight'][0] == (k + 1, a.embed_dim) and spec[p + 'embed_ema'][0] == (k, a.embed_dim)
        assert spec[p + 'cluster_size_ema'][0] == (k,)
        assert torch.equal(sd[p + 'embed_ema'], sd[p + 'weight'][:-1]) and not sd[p + 'weight'][-1].any()
    shared = {'quantizer.codebooks.%d' % d: 'quantizer.codebooks.0' for d in range(1, D)} if a.shared_codebook else {}
    assert spec.module_aliases == shared
    assert (sd['quantizer.codebooks.%d.weight' % (D - 1)].data_ptr() == sd['quantizer.codebooks.0.weight'].data_ptr()) \
        == (a.shared_codebook or D == 1)

    eng, _ = repacked(cls, a, spec)
    assert [eng._n_embed(d) for d in range(D)] == list(a.n_embeds)
    rec = install(monkeypatch)
    ks, call = [], rec.call

    def record(name, args):
        if name in ('l2_argmin_tc', 'l2_argmin_tc_split'):
            ks.append((args['K'], args['pack'][0].shape[0], args['codebook'].shape[0]))
        call(name, args)
    rec.call = record
    z = torch.rand(64, a.embed_dim, generator=torch.Generator().manual_seed(0))
    calls = _calls(model, eng, *SIZES[model]) + [('quantize', lambda: eng.quantize(z))]
    if len(set(a.n_embeds)) == 1:                           # the models' get_soft_codes takes codebooks of one size
        calls.append(('soft_codes', lambda: eng.soft_codes(z, 1.0)))
    for label, thunk in calls:
        n = len(ks)
        thunk()
        if len(ks) > n:                                     # one argmin per depth, in depth order
            assert [k for k, _, _ in ks[n:]] == list(a.n_embeds), label
            assert all(pk == k and rows >= k + 1 for k, pk, rows in ks[n:]), label
    assert ks
