"""fastfp_b200 -- an H100-native engine for the pulsar-timing Fp-statistic frequency scan.

Drop-in for the hot path of gabefreedman/fastfp (``FastFp.calculate_Fp``, ``NMFP.calculate_nmfp``,
``fastfp.utils.get_xCy``): same Python call signatures, with the JAX/XLA kernels replaced by
hand-written fp64 CUDA kernels for sm_90a behind a C ABI (``include/fastfp_b200.h``).
"""
from .blockn import BlockNvec
from .fastfp import FastFp
from .fe import FastFe
from .nmfp import NMFP, CURN_container, GPEcorr_container, RN_container
from . import chains, model  # noqa: F401
from .model import setup_fp_model
from .utils import compute_sigmas, compute_TNTs, get_mats_fp, get_mats_nmfp, get_xCy
from .vmap import vmap

__version__ = "0.1.0"
__all__ = ["BlockNvec", "FastFp", "FastFe", "NMFP", "RN_container", "CURN_container", "GPEcorr_container", "get_xCy", "get_mats_fp",
           "get_mats_nmfp", "compute_TNTs", "compute_sigmas", "vmap", "setup_fp_model"]
