"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's residual quantiser at any depth D
(RQBottleneck.quantize / compute_commitment_loss / embed_code / embed_code_with_depth / embed_partial_code /
get_soft_codes, `archs/tdcrqvae3_arch.py:294-457`) over a list of D codebook weights [K + 1, E] (the same tensor D
times for a shared codebook).  Only tests/ import it; it is pinned against outputs of the reference's own methods
(tests/golden/rq_*.pt, minted by `python -m oracle.make_rq_golden`).  At D = 1 it computes what oracle/pgt_oracle.py and
oracle/codec_oracle.py compute."""
import torch
import torch.nn.functional as F

from oracle.pgt_oracle import l2_distances


def codebooks(sd, depth):
    """The D codebook weights of a state dict, in depth order."""
    return [sd['quantizer.codebooks.%d.weight' % d] for d in range(depth)]


def quantize(cbs, x):
    """RQBottleneck.quantize + compute_commitment_loss (`:294-352`) of x [..., E] fp32 ->
    (quant_list: the aggregate after each depth, codes [..., D] int64, loss)."""
    residual = x.detach().clone()
    agg = torch.zeros_like(x)
    quant_list, code_list = [], []
    for cb in cbs:
        code = l2_distances(cb, residual).argmin(dim=-1)
        quant = F.embedding(code, cb)
        residual.sub_(quant)
        agg.add_(quant)
        quant_list.append(agg.clone())
        code_list.append(code.unsqueeze(-1))
    loss = torch.mean(torch.stack([(x - q).pow(2.0).mean() for q in quant_list]))
    return quant_list, torch.cat(code_list, dim=-1), loss


def embed_with_depth(cbs, code):
    """embed_code_with_depth (`:371-391`): codes [..., D] -> [..., D, E], not summed."""
    return torch.stack([F.embedding(code[..., d], cb) for d, cb in enumerate(cbs)], dim=-2)


def embed_code(cbs, code):
    """embed_code (`:355-368`): the depth sum of the code rows."""
    return embed_with_depth(cbs, code).sum(-2)


def embed_partial(cbs, code, code_idx, decode_type):
    """embed_partial_code (`:394-426`): 'select' -> depth code_idx's rows, 'add' -> the sum over depths 0..code_idx."""
    e = embed_with_depth(cbs, code)
    if decode_type == 'select':
        return e[..., code_idx, :]
    return e[..., :code_idx + 1, :].sum(-2)


def soft_codes(cbs, x, temp):
    """get_soft_codes, stochastic=False (`:429-457`): softmax(-dist / temp) of each depth's residual ->
    (soft codes [..., D, K], codes [..., D])."""
    residual = x.detach().clone()
    soft, codes = [], []
    for cb in cbs:
        d = l2_distances(cb, residual)
        soft.append(F.softmax(-d / temp, dim=-1).unsqueeze(-2))
        code = d.argmin(dim=-1)
        residual -= F.embedding(code, cb)
        codes.append(code.unsqueeze(-1))
    return torch.cat(soft, dim=-2), torch.cat(codes, dim=-1)
