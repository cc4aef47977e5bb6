"""CUDA-graph replay of the registered models' calls (model.cuda_graph -> Engine.graphed): VQAutoEncoder, CodeFormer,
RQVAE, TDRQVAE and TDCRQVAE3.

Each replayed call gives the eager bits (outputs, losses and statistics alike) on two inputs of one shape and on a
second shape, which gets a capture of its own; a replay issues no launch through the C ABI (the launch counter stays
put); a replay's outputs are the graph's static tensors, which a following eager call leaves alone.  Then the
VQAutoEncoder code counts, the scratch memory a capture takes (the graph's own, not the process-wide workspace cache),
the weights a replay reads after load_state_dict(), the host-side argument checks in graph
mode, and PGTFormer, whose cuda_graph keeps covering its forward alone.  The unmarked tests at the top need no GPU."""
import copy

import pytest
import torch

DEV = 'cuda'
FIVE = ('VQAutoEncoder', 'CodeFormer', 'RQVAE', 'TDRQVAE', 'TDCRQVAE3')


def _config(name, network_g):
    """Constructor arguments of each registered model: the synthetic configurations of the models' own tests."""
    from oracle.make_rqvae_golden import CONFIGS
    if name in ('VQAutoEncoder', 'CodeFormer'):
        return {}
    g = copy.deepcopy(CONFIGS['r2']) if name == 'RQVAE' else copy.deepcopy(network_g)
    g.pop('type', None)
    return g


def _build(name, network_g):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    return ARCH_REGISTRY.get(name)(**_config(name, network_g))


# --------------------------------------------------------------------------- without a GPU
def test_every_registered_model_has_cuda_graph(network_g, monkeypatch):
    """cuda_graph is off on the five models even with PGT_CUDA_GRAPH=1, which keeps turning on PGTFormer's forward."""
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    assert set(ARCH_REGISTRY.keys()) == set(FIVE) | {'PGTFormer'}
    monkeypatch.setenv('PGT_CUDA_GRAPH', '1')
    for name in FIVE:
        m = _build(name, network_g)
        assert m.cuda_graph is False, name
        del m
    assert _build('PGTFormer', network_g).cuda_graph is True
    monkeypatch.setenv('PGT_CUDA_GRAPH', '0')
    assert _build('PGTFormer', network_g).cuda_graph is False


@pytest.mark.parametrize('shape', [(2, 3, 64, 64), (3, 3, 48, 64), (3, 4, 64, 64), (3, 64, 64)])
def test_tdcrqvae3_forward_checks_frames_first(network_g, shape):
    """TDCRQVAE3.forward / get_codes check their frames on the host, before the engine (here: before the missing
    CUDA device) is reached, so a graphed call never starts a warm-up or capture on a bad input."""
    m = _build('TDCRQVAE3', network_g)
    m.cuda_graph = True
    for call in (m, m.get_codes):
        with pytest.raises(ValueError):
            call(torch.rand(*shape))


# --------------------------------------------------------------------------- replay against eager
_models = {}


def model_of(name, network_g):
    if name not in _models:
        _models[name] = _build(name, network_g).to(DEV).eval()
    return _models[name]


def rand(*shape, seed, lo=0.0, hi=1.0):
    return (torch.rand(*shape, generator=torch.Generator().manual_seed(seed)) * (hi - lo) + lo).to(DEV)


def codes(m, F, h, w, seed):
    """Integer codes [F, h, w, D], each depth's in [0, n_embed_d] (its padding row included)."""
    D = m.code_shape[-1]
    n = list(getattr(m.arch, 'n_embeds', None) or [m.arch.n_embed] * D)
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, k + 1, (F, h, w), generator=g) for k in n], -1).to(DEV)


def flat(o):
    if torch.is_tensor(o):
        return [o]
    if isinstance(o, dict):
        return [t for k in sorted(o) for t in flat(o[k])]
    if isinstance(o, (tuple, list)):
        return [t for v in o for t in flat(v)]
    return []


def same_bits(got, ref):
    got, ref = flat(got), flat(ref)
    assert len(got) == len(ref) and got
    for a, b in zip(got, ref):
        assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)


def clone(o):
    return [t.clone() for t in flat(o)]


def check_replay(m, call, same, other):
    """call(*args) is one model call; same: two argument tuples of one shape; other: one of another shape."""
    from pgtformer_b200 import ops
    m.cuda_graph = False
    refs = [clone(call(*a)) for a in same + [other]]
    m.cuda_graph = True
    try:
        same_bits(call(*same[0]), refs[0])                     # warm-up, capture, first replay
        n = ops.launch_count()
        got = call(*same[1])
        assert ops.launch_count() == n                         # a replay: no launch through the C ABI
        same_bits(got, refs[1])
        kept = clone(got)
        m.cuda_graph = False
        call(*same[0])
        same_bits(got, kept)                                   # the static outputs outlive an eager call
        m.cuda_graph = True
        same_bits(call(*other), refs[2])                       # a second shape: its own capture
        n = ops.launch_count()
        same_bits(call(*same[0]), refs[0])                     # the first graph still replays
        assert ops.launch_count() == n
        assert not torch.cuda.is_current_stream_capturing()
    finally:
        m.cuda_graph = False


def _img(b, H, seed, lo=0.0):
    return (rand(b, 3, H, H, seed=seed, lo=lo),)


CASES = {
    # VQAutoEncoder: 128^2 images (a 4 x 4 latent), both code_only values
    ('VQAutoEncoder', 'forward'): (lambda m, x: m(x), lambda m, b, s: _img(b, 128, s, -1.0)),
    ('VQAutoEncoder', 'forward_code_only'): (lambda m, x: m(x, code_only=True), lambda m, b, s: _img(b, 128, s, -1.0)),
    # CodeFormer: 512^2 only; the key holds w, adain and code_only
    ('CodeFormer', 'forward_w05_adain'): (lambda m, x: m(x, w=0.5, adain=True), lambda m, b, s: _img(b, 512, s, -1.0)),
    ('CodeFormer', 'forward_w0'): (lambda m, x: m(x, w=0, adain=False), lambda m, b, s: _img(b, 512, s, -1.0)),
    ('CodeFormer', 'forward_code_only'): (lambda m, x: m(x, w=0.5, code_only=True),
                                          lambda m, b, s: _img(b, 512, s, -1.0)),
    # RQVAE R2: 64^2 images (an 8 x 8 latent of 3 depths with codebooks of 512, 1024 and 256 codes)
    ('RQVAE', 'forward'): (lambda m, x: m(x), lambda m, b, s: _img(b, 64, s)),
    ('RQVAE', 'forward_code_only'): (lambda m, x: m(x, code_only=True), lambda m, b, s: _img(b, 64, s)),
    ('RQVAE', 'get_codes'): (lambda m, x: m.get_codes(x), lambda m, b, s: _img(b, 64, s)),
    ('RQVAE', 'get_codesbt'): (lambda m, x: m.get_codesbt(x), lambda m, b, s: (rand(1, b + 1, 3, 64, 64, seed=s),)),
    ('RQVAE', 'encode'): (lambda m, x: m.encode(x), lambda m, b, s: _img(b, 64, s)),
    ('RQVAE', 'decode'): (lambda m, z: m.decode(z), lambda m, b, s: (rand(b, 8, 8, 128, seed=s, lo=-1.0),)),
    ('RQVAE', 'decode_code'): (lambda m, c: m.decode_code(c), lambda m, b, s: (codes(m, b, 8, 8, s),)),
    # TDRQVAE: clips of 3 frames of 64^2
    ('TDRQVAE', 'forward'): (lambda m, x: m(x), lambda m, b, s: (rand(b, 3, 3, 64, 64, seed=s),)),
    ('TDRQVAE', 'forward_code_only'): (lambda m, x: m(x, code_only=True), lambda m, b, s: (rand(b, 3, 3, 64, 64, seed=s),)),
    ('TDRQVAE', 'get_codes'): (lambda m, x: m.get_codes(x), lambda m, b, s: (rand(b, 3, 3, 64, 64, seed=s),)),
    ('TDRQVAE', 'get_codesbt'): (lambda m, x: m.get_codesbt(x), lambda m, b, s: (rand(b, 3, 3, 64, 64, seed=s),)),
    ('TDRQVAE', 'encode'): (lambda m, x: m.encode(x), lambda m, b, s: _img(3 * b, 64, s)),
    ('TDRQVAE', 'decode'): (lambda m, z: m.decode(z),
                            lambda m, b, s: (rand(3 * b, 4, 4, m.arch.embed_dim, seed=s, lo=-1.0),)),
    ('TDRQVAE', 'decode_code'): (lambda m, c: m.decode_code(c), lambda m, b, s: (codes(m, 3 * b, 4, 4, s),)),
    # TDCRQVAE3: 3-frame clips of 64^2 as frames [3b, 3, 64, 64]
    ('TDCRQVAE3', 'forward'): (lambda m, x: m(x), lambda m, b, s: _img(3 * b, 64, s)),
    ('TDCRQVAE3', 'forward_code_only'): (lambda m, x: m(x, code_only=True), lambda m, b, s: _img(3 * b, 64, s)),
    ('TDCRQVAE3', 'get_codes'): (lambda m, x: m.get_codes(x), lambda m, b, s: _img(3 * b, 64, s)),
    ('TDCRQVAE3', 'encode'): (lambda m, x: m.encode(x), lambda m, b, s: _img(3 * b, 64, s)),
    ('TDCRQVAE3', 'decode'): (lambda m, z: m.decode(z),
                              lambda m, b, s: (rand(3 * b, 4, 4, m.arch.embed_dim, seed=s, lo=-1.0),)),
    ('TDCRQVAE3', 'decode_code'): (lambda m, c: m.decode_code(c), lambda m, b, s: (codes(m, 3 * b, 4, 4, s),)),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name,call', sorted(CASES), ids=['%s-%s' % k for k in sorted(CASES)])
def test_replay_matches_eager(network_g, name, call):
    m = model_of(name, network_g)
    fn, make = CASES[name, call]
    check_replay(m, lambda *a: fn(m, *a), [make(m, 1, 1), make(m, 1, 2)], make(m, 2, 3))


# --------------------------------------------------------------------------- VQAutoEncoder code counts
@pytest.mark.gpu
def test_vqgan_usage_graphed_equals_eager(network_g):
    """A replay adds its counts to the usage buffer the module holds at call time: eager, eager, reset_usage(), eager
    and the same sequence graphed leave the same counts, before and after the reset."""
    m = model_of('VQAutoEncoder', network_g)
    xs = [_img(1, 128, s, -1.0)[0] for s in (4, 5, 6)]

    def run(graph):
        m.cuda_graph = graph
        try:
            q = m.quantize
            q.reset_usage()
            m(xs[0])
            m(xs[1])
            before = q.usage.clone()
            q.reset_usage()
            m(xs[2])
            return before, q.usage.clone()
        finally:
            m.cuda_graph = False

    eager, graphed = run(False), run(True)
    assert int(eager[0].sum()) == 2 * 16 and int(eager[1].sum()) == 16       # 16 latent tokens per 128^2 image
    assert torch.equal(graphed[0], eager[0]) and torch.equal(graphed[1], eager[1])


# --------------------------------------------------------------------------- scratch memory of a capture
@pytest.mark.gpu
def test_captured_scratch_belongs_to_the_graph(network_g):
    """The GroupNorm scratch a capture uses comes from that graph's pool, never from the process-wide workspace cache:
    a graph captured after another graph was destroyed, and kept while a larger key is captured, replays the eager bits,
    and no cached workspace is keyed by a capture stream."""
    from pgtformer_b200 import ops
    m = _build('RQVAE', network_g).to(DEV).eval()
    small, large = _img(1, 64, 12)[0], _img(8, 128, 13)[0]
    ref_small, ref_large = clone(m(small)), clone(m(large))
    before = {k: v.data_ptr() for k, v in ops._gn_ws.items()}
    m.cuda_graph = True
    try:
        m(small)
        streams = [m.engine().capture_stream.cuda_stream]
        m.refresh()                                            # destroys that graph and its pool
        torch.cuda.empty_cache()
        same_bits(m(small), ref_small)                         # the same key, captured again
        same_bits(m(large), ref_large)                         # a key that needs more scratch
        streams.append(m.engine().capture_stream.cuda_stream)
        # (a stream handle may be recycled from an earlier test: only entries made or changed since count)
        assert all(before.get(k) == v.data_ptr() for k, v in ops._gn_ws.items() if k[2] in streams)
        m.cuda_graph = False
        m(large)
        torch.cuda.empty_cache()
        m.cuda_graph = True
        same_bits(m(small), ref_small)
        same_bits(m(large), ref_large)
    finally:
        m.cuda_graph = False


# --------------------------------------------------------------------------- stale weights
@pytest.mark.gpu
def test_replay_reads_the_loaded_weights(network_g):
    """load_state_dict() drops the engine and its graphs: the next graphed call runs on the new weights."""
    m = _build('RQVAE', network_g).to(DEV).eval()
    x = _img(1, 64, 7)[0]
    m.cuda_graph = True
    old = clone(m(x))
    sd = {k: v * 0.9 if v.is_floating_point() else v for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    got = clone(m(x))
    m.cuda_graph = False
    same_bits(got, m(x))
    assert not torch.equal(got[0], old[0])


# --------------------------------------------------------------------------- host-side checks in graph mode
@pytest.mark.gpu
def test_bad_arguments_raise_before_any_capture(network_g):
    m = model_of('RQVAE', network_g)
    x = _img(1, 64, 8)[0]
    c = codes(m, 1, 8, 8, 9)
    m.cuda_graph = False
    ref_x, ref_c = clone(m(x)), clone(m.decode_code(c))
    m.cuda_graph = True
    try:
        with pytest.raises(ValueError):
            m(rand(1, 3, 64, 100, seed=1))
        with pytest.raises(ValueError):
            m.decode_code(c[..., :2])
        bad = c.clone()
        bad[0, 0, 0, 2] = m.arch.n_embeds[2] + 1
        with pytest.raises(IndexError):
            m.decode_code(bad)
        assert not torch.cuda.is_current_stream_capturing()
        same_bits(m(x), ref_x)
        same_bits(m.decode_code(c), ref_c)
    finally:
        m.cuda_graph = False


# --------------------------------------------------------------------------- PGTFormer keeps its forward-only graphs
@pytest.mark.gpu
def test_pgtformer_codec_calls_stay_eager(network_g):
    from pgtformer_b200 import ops
    m = _build('PGTFormer', network_g).to(DEV).eval()
    m.cuda_graph = True
    x1, x2 = _img(3, 64, 10)[0], _img(3, 64, 11)[0]
    c1 = m.get_codes(x1)
    kept = c1.clone()
    n = ops.launch_count()
    c2 = m.get_codes(x2)
    assert ops.launch_count() > n and torch.equal(c1, kept) and c1.data_ptr() != c2.data_ptr()
    d1 = m.decode_code(c1)
    kept = d1.clone()
    n = ops.launch_count()
    d2 = m.decode_code(c2)
    assert ops.launch_count() > n and torch.equal(d1, kept) and d1.data_ptr() != d2.data_ptr()
    assert not getattr(m.engine(), '_graphs', None)
