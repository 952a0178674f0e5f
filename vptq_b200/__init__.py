"""vptq_b200: the VPTQ quantized-linear hot path, written from scratch for NVIDIA H100 (sm_90a).

Public surface = the reference's (vptq/__init__.py:7-15): `VQuantLinear`, `ops`, `__version__`.
"""
from . import ops
from .fuse import fuse, set_batched_decode, set_list_decode, set_lists_prefill, set_quant_grad, unfuse
from .layers import VQuantLinear

# Hugging Face gates its VPTQ integration on the installed `vptq` version being >= 0.0.4
# (transformers/utils/import_utils.py); this build speaks that surface.
__version__ = "0.0.5+b200"

__all__ = ["VQuantLinear", "ops", "fuse", "unfuse", "set_quant_grad", "set_batched_decode", "set_lists_prefill",
           "set_list_decode", "__version__"]
