"""go-ibft_b200 -- H100 (sm_90a) batched message-verification engine behind go-ibft's core.Verifier / core.Messages.

Only the hot path of SURVEY.md §8 lives here: csrc/ (hand-written sm_90a CUDA kernels + the C ABI of
include/ibft_verify.h) and the host-side mirror of the reference interfaces for that path.
"""
from .engine import (Engine, EngineError, GROUP_DTYPE, ITEM_DTYPE, KIND_DIGEST, KIND_INVALID, KIND_PAYLOAD, KIND_SEAL,  # noqa: F401
                     KIND_WIRE, KIND_WIRE_SEAL, KIND_PAYLOAD2, ITEM_OK, ITEM_NEEDS_HOST,
                     NO_TABLE, PROPOSER_NONE, PROPOSER_UNSET, QUORUM_DEFAULT, QUORUM_PREPARE, QUORUM_PREPREPARE, RESULT_DTYPE,
                     group_descs, load_library)
