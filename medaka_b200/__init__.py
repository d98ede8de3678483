"""medaka_b200: a Hopper (sm_90a) engine for medaka's consensus-inference hot path.

Python here is the host-side mirror of the reference's interface for that path
(Sample / Region / CountsFeatureEncoder / Batch / GRUModel.predict_on_batch /
HaploidLabelScheme.decode_consensus / run_prediction); all arithmetic runs in
libmedaka_b200.so (hand-written CUDA, C ABI in include/medaka_b200.h).  There is no
CPU fallback: without the library, or without an H100, calls raise.
"""
__version__ = "0.1.0"
