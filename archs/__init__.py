from .pgtformer_arch import PGTFormer, TDCRQVAE3  # noqa: F401
from .tdrqvae_arch import TDRQVAE  # noqa: F401
