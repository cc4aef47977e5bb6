"""TEST INFRASTRUCTURE ONLY — CPU restatement of the stage-I codec methods of the reference's TDCRQVAE3
(`archs/tdcrqvae3_arch.py:774-813`, RQBottleneck.get_soft_codes :429-457) on top of the forward-path restatement in
oracle/pgt_oracle.py.  Like that module it is the checker: only tests/ import it; it is pinned against outputs of the
reference's own methods (tests/golden/tdcrqvae3_codec_*.pt, minted by `python -m oracle.make_codec_golden`)."""
import torch.nn.functional as F

from oracle.pgt_oracle import conv, decoder_forward, encoder_forward, l2_distances


def tdcrqvae3_encode(sd, arch, x):
    """TDCRQVAE3.encode (`archs/tdcrqvae3_arch.py:774-777`): quant_conv(Encoder(x)) as NHWC [b*3, H/16, W/16, E]."""
    h, _ = encoder_forward(sd, arch, x)
    return conv(sd, 'quant_conv', h).permute(0, 2, 3, 1).contiguous()


def tdcrqvae3_decode(sd, arch, z_q):
    """TDCRQVAE3.decode (`archs/tdcrqvae3_arch.py:779-783`): NHWC z_q -> post_quant_conv -> Decoder.forward."""
    return decoder_forward(sd, arch, conv(sd, 'post_quant_conv', z_q.permute(0, 3, 1, 2).contiguous()))


def soft_codes(codebook_weight, z, temp):
    """RQBottleneck.get_soft_codes, depth 1, stochastic=False (`archs/tdcrqvae3_arch.py:429-457`): softmax over the
    fp32 addmm distances (padding row excluded) -> (soft_code [..., 1, K], code [..., 1] = first-minimum argmin)."""
    d = l2_distances(codebook_weight, z)
    return F.softmax(-d / temp, dim=-1).unsqueeze(-2), d.argmin(dim=-1).unsqueeze(-1)
