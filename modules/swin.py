"""Drop-in `modules/swin.py::BasicLayer` (the Video-Swin stage the reference's TDRQVAE wraps around its quantiser,
`archs/tdrqvae_arch.py:30,834-835`): same import path, constructor keywords, state-dict names and
`forward(x[B, C, D, H, W]) -> [B, C, D, H, W]` as the reference's `modules/swin.py:326-405`, running on the H100
kernels (pgtformer_b200/swin3d.py).  Inference only; no CPU path."""
from pgtformer_b200.swin3d import BasicLayer  # noqa: F401
