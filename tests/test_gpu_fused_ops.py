"""The fused linear combinations of the group law (secp_fe.cuh) on the device -- the PTX carry chains -- against big integers,
at the carry and borrow edges of tests/fused_edges.py, through ibft_debug_op (IBFT_DBG_FE_FUSED)."""
import pytest

import fused_edges as FE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import ibft_b200 as ib
    e = ib.Engine(device=0)
    yield e
    e.close()


def test_fused_ops_match_big_integers(dev):
    cs = FE.cases()
    res = dev.debug_op("FE_FUSED", [a for _, a, _, _ in cs], [b for _, _, b, _ in cs], [FE.c_operand(s, c) for s, _, _, c in cs])
    bad = FE.check(res, cs)
    assert not bad, "\n".join(bad[:20])
