"""H100 launch sequence of the registered RQVAE (`archs/rqvae_arch.py:779-931`): TDRQVAE's 2-D Encoder / Decoder with
dense AttnBlocks, walked by Engine from the arch's block lists, around the residual quantiser of Engine.quantize, over
libpgt_b200.so.

Separate codebooks may differ in size.  They are stacked once, each padded to the largest K + 1 rows, so that rq_embed
reads every depth's rows (the padding row of depth d stays at index K_d) and the argmin of depth d scans its own K_d
codes.  The argmins run split over code ranges (ops.l2_argmin_tc_split): RQ-VAE latents are small (64 tokens per 256^2
image at f = 32), so the unsplit sweep would scan each large codebook on a handful of SMs.  Every op is a call into the
C ABI; there is no PyTorch / CPU fallback."""
from . import ops
from .engine import Engine
from .spec import RQVAEArch


class RQVAEEngine(Engine):
    arch_class = RQVAEArch

    def _argmin(self, *a, **k):
        return ops.l2_argmin_tc_split(*a, **k)
