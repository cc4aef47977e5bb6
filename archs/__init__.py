from .pgtformer_arch import PGTFormer, TDCRQVAE3  # noqa: F401
from .tdrqvae_arch import TDRQVAE  # noqa: F401
from .vqgan_arch import VQAutoEncoder  # noqa: F401
from .codeformer_arch import CodeFormer  # noqa: F401
