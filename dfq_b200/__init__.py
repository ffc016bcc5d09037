"""dfq_b200: H100-native (sm_90a) implementation of the DFQ calibration hot path.

Cross-layer weight equalization, bias correction, BN folding and fake quantization of
jakc4103/DFQ, computed by hand-written CUDA kernels behind a C ABI (include/dfq_b200.h).
The modules mirror the reference's own entry points:

    dfq_b200.dfq                     <- dfq.py
    dfq_b200.utils.quantize          <- utils/quantize.py
    dfq_b200.utils.layer_transform   <- utils/layer_transform.py
    dfq_b200.utils.relation          <- utils/relation.py
    dfq_b200.improve_dfq             <- improve_dfq.py (update_quant_range / set_update_stat)

There is no CPU implementation in this package: without a CUDA device the tensor functions raise.
"""
__version__ = "0.1.0"
