"""rl4co_b200 -- H100 (sm_90a) rollout engine behind rl4co's env / decoder API.

Scope: the autoregressive construction hot path only (SURVEY.md section 8):
  envs      FusedTSPEnv, FusedCVRPEnv          <- rl4co.envs.TSPEnv / CVRPEnv
  decoder   FusedAttentionModelDecoder         <- rl4co.models.zoo.am.decoder
  policy    FusedAttentionModelPolicy          <- rl4co.models.zoo.am.policy (loop owner)
  polynet   FusedPolyNetPolicy, polynet_step   <- rl4co.models.zoo.polynet (AM encoder)
  decoding  Greedy / Sampling / Evaluate       <- rl4co.utils.decoding
  native    ctypes binding of libcorollout.so  (include/corollout.h)
"""

from .tensordict import TensorDict  # noqa: F401

__version__ = "0.1.0"
__all__ = ["TensorDict", "FusedTSPEnv", "FusedCVRPEnv", "FusedAttentionModelDecoder", "FusedAttentionModelPolicy",
           "FusedPolyNetDecoder", "FusedPolyNetPolicy", "polynet_step", "get_env"]


def __getattr__(name):  # lazy: importing the package must not require the CUDA library
    if name in ("FusedTSPEnv", "FusedCVRPEnv", "get_env", "TSPGenerator", "CVRPGenerator"):
        from . import envs

        return getattr(envs, name)
    if name in ("FusedAttentionModelDecoder", "FusedPrecomputedCache"):
        from . import decoder

        return getattr(decoder, name)
    if name in ("FusedAttentionModelPolicy", "AttentionModelPolicy"):
        from . import policy

        return getattr(policy, name)
    if name in ("FusedPolyNetDecoder", "FusedPolyNetPolicy", "PolyNetPolicy", "polynet_step"):
        from . import polynet

        return getattr(polynet, name)
    raise AttributeError(name)
