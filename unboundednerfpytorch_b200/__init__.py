"""unboundednerfpytorch_b200 -- H100-native (sm_90a) volumetric-rendering hot path for the FourierGrid / DVGO
models of sjtuytc/UnboundedNeRFPytorch, behind the reference's own extension / autograd / module surface.

Layout: ``csrc/`` hand-written CUDA + the C ABI (include/ubnerf_b200.h) -> ``libubnerf_b200.so``;
``_cabi`` ctypes binding; ``ops`` the four legacy extension modules' functions; ``functional`` Raw2Alpha /
Alphas2Weights; ``grid`` DenseGrid / FourierGrid / MaskGrid; ``masked_adam`` MaskedAdam; ``march`` the fused
per-ray kernel; ``models`` FourierGridModel / DirectContractedVoxGO; ``dist`` ray sharding over NCCL.
There is no CPU / eager fallback: without the built library every op raises.
"""
from . import _cabi  # noqa: F401

__version__ = '0.1.0'


def install_legacy_modules():
    """Register render_utils_cuda / total_variation_cuda / adam_upd_cuda / ub360_utils_cuda in sys.modules."""
    from . import legacy
    return legacy.install()
