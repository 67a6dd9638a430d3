"""racinglmpc_b200 — H100-native (sm_90a) batched LMPC finite-time optimal control (drop-in for the
urosolia/RacingLMPC hot path).  See DESIGN.md / INTEGRATION.md."""
from .batched import BatchedFTOCP, pack_abc  # noqa: F401

__all__ = ["BatchedFTOCP", "pack_abc"]
