"""The block lists the engines walk and the state-dict layouts the spec builders write agree beyond the configurations
of the reference fixtures: over a grid of configurations of the six registered models, run on the CPU with every kernel
call replaced by test_walk_cpu's recorder, every `encoder.` / `decoder.` / `generator.` block the spec declares is read
by some call, and no call looks up a weight the spec does not declare."""
import copy
import re

import pytest

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


# (model, id, top-level overrides, ddconfig overrides), TDCRQVAE3 / PGTFormer / TDRQVAE on the options file's network_g,
# RQVAE on the R2 fixture configuration, VQGAN and CodeFormer on their constructor defaults
GRID = [('TDCRQVAE3', 'r%d' % r, {}, {'num_res_blocks': r}) for r in (1, 2, 3)] + \
    [('TDCRQVAE3', 'attn%d' % len(a), {}, {'attn_resolutions': a}) for a in ([], [32], [32, 64])] + \
    [('TDCRQVAE3', 'levels%d' % len(m), {}, _levels(*m)) for m in ((1, 2, 4), (1, 2, 4, 8), (1, 1, 2, 4, 4, 8))] + \
    [('TDCRQVAE3', 'd%d_%s' % (d, 'shared' if s else 'separate'), _rq(d, s, 32), {})
     for d in (1, 2, 4) for s in (True, False)] + \
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
    [('RQVAE', 'r%d' % r, {}, {'num_res_blocks': r}) for r in (1, 3)] + \
    [('VQGAN', 'res_blocks%d' % r, {'res_blocks': r}, {}) for r in (1, 3)] + \
    [('VQGAN', 'levels4', {'ch_mult': [1, 2, 2, 4], 'attn_resolutions': [64]}, {})] + \
    [('CodeFormer', 'connect_' + ('_'.join(c) or 'none'), {'connect_list': c}, {})
     for c in ([], ['32'], ['16', '512'], ['64', '128', '256'], ['16', '32', '64', '128', '256', '512'])]

SIZES = {'TDCRQVAE3': (1, 128, 128), 'PGTFormer': (1, 64, 64), 'TDRQVAE': (1, 128, 128), 'RQVAE': (1, 128, 128),
         'VQGAN': (1, 128, 128), 'CodeFormer': (1, 512, 512)}


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
    if model == 'RQVAE':
        from oracle.make_rqvae_golden import CONFIGS
        g = copy.deepcopy(CONFIGS['r2'])
    else:
        g = copy.deepcopy(network_g)
    g.update(top)
    g['ddconfig'].update(dd)
    if model == 'TDRQVAE':
        return (TDRQVAEEngine, *S.build_tdrqvae_spec(dict(g, type='TDRQVAE')))
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
