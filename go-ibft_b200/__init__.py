"""go-ibft_b200 -- H100 (sm_90a) batched message-verification engine behind go-ibft's core.Verifier / core.Messages.

Only the hot path of SURVEY.md §8 lives here: csrc/ (hand-written sm_90a CUDA kernels + the C ABI of
include/ibft_verify.h) and the host-side mirror of the reference interfaces for that path.
"""
from .engine import (Engine, EngineError, GROUP_DTYPE, ITEM_DTYPE, KIND_DIGEST, KIND_INVALID, KIND_PAYLOAD, KIND_SEAL,  # noqa: F401
                     KIND_WIRE, KIND_WIRE_SEAL, KIND_PAYLOAD2, ITEM_OK, ITEM_NEEDS_HOST,
                     NO_TABLE, PROPOSER_NONE, PROPOSER_UNSET, QUORUM_DEFAULT, QUORUM_PREPARE, QUORUM_PREPREPARE, RESULT_DTYPE,
                     REASON_BAD_V, REASON_INCONSISTENT, REASON_MALFORMED, REASON_NEEDS_HOST, REASON_NO_GROUP, REASON_NO_KEY,
                     REASON_NOT_VALIDATOR, REASON_OK, REASON_R_NOT_X, REASON_R_RANGE, REASON_S_RANGE, REASON_SIGNER_MISMATCH,
                     group_descs, load_library,
                     GROUP_HASH_DTYPE, HASH_COMMIT, HASH_PREPARE, HASH_UNBOUND, group_hashes)
