"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's registered RQVAE (`archs/rqvae_arch.py:779-931`),
functional on a state dict.  Only tests/ import it; it is pinned against the outputs of the reference's own module
(tests/golden/rqvae_*.pt, minted by `python -m oracle.make_rqvae_golden`).

Nothing is restated here: the Encoder / Decoder (`:579-776`) are TDRQVAE's (oracle/tdrqvae_oracle.py: ResnetBlock,
AttnBlock, Downsample with the (0, 1, 0, 1) pad, nearest Upsample + conv) and the RQBottleneck (`:324-575`) is
oracle/rq_oracle.py's, whose per-depth codebook list takes separate codebooks of different sizes as they are."""
from oracle import rq_oracle as RQ
from oracle.tdrqvae_oracle import decode, encode


def codebooks(sd, arch):
    return RQ.codebooks(sd, arch.depth)


def forward(sd, arch, x, code_only=False):
    """RQVAE.forward (`:828-834`) of x [B,3,H,W]: (out [B,3,H,W] or, code_only, z_q [B,h,w,E], quant_loss,
    code [B,h,w,D]).  z_q is x + (q - x), the straight-through value the reference returns (`:453-454`)."""
    z_e = encode(sd, arch, x)
    quant_list, code, loss = RQ.quantize(codebooks(sd, arch), z_e)
    z_q = z_e + (quant_list[-1] - z_e)
    if code_only:
        return z_q, loss, code
    return decode(sd, arch, z_q), loss, code


def decode_code(sd, arch, code):
    """RQVAE.decode_code (`:868-872`): the depth sum of the code rows, decoded."""
    return decode(sd, arch, RQ.embed_code(codebooks(sd, arch), code))


def decode_partial_code(sd, arch, code, code_idx, decode_type='select'):
    """RQVAE.decode_partial_code (`:913-922`)."""
    return decode(sd, arch, RQ.embed_partial(codebooks(sd, arch), code, code_idx, decode_type))


def get_soft_codes(sd, arch, xs, temp=1.0):
    """RQVAE.get_soft_codes (`:860-866`), stochastic=False: (soft codes [B,h,w,D,K], codes [B,h,w,D])."""
    return RQ.soft_codes(codebooks(sd, arch), encode(sd, arch, xs), temp)
