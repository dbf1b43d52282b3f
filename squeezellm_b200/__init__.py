"""squeezellm_b200 - H100-native (sm_90a) drop-in for SqueezeLLM's dense-and-sparse LUT-GEMV hot path.

Public surface (mirrors the reference's squeezellm/quant.py):
    QuantLinearLUT, make_quant_lut, round_to_nearest_pole_sim      -> squeezellm_b200.quant
    quant_cuda                                                    -> the compiled extension (12 reference symbols + lutgemv_fused)
    SiblingGroup, fuse_siblings                                   -> squeezellm_b200.fusion   (q/k/v, gate/up as one launch)
    load_quantized, quantized_state_dict                          -> squeezellm_b200.checkpoint (reference checkpoints in / out)
    GraphedDecodeStep                                             -> squeezellm_b200.runtime
    shard_bounds, shard_state, ShardedQuantLinearLUT, PeerExchange -> squeezellm_b200.sharding
Importing `squeezellm_b200.quant` requires the compiled extension (no CPU fallback).
"""
__version__ = "0.1.0"


def __getattr__(name):  # lazy: `import squeezellm_b200` alone must not need torch or the extension
    if name in ("QuantLinearLUT", "make_quant_lut", "round_to_nearest_pole_sim", "pack_indices", "quant_cuda"):
        from . import quant as _q
        return getattr(_q, name)
    raise AttributeError(name)
