"""The arithmetic edge sweep of tests/arith_edges.py on the device (the PTX carry-chain paths), through ibft_debug_op on one
engine built here, and the same sweep against builds of engine.cu with each opt-in field-arithmetic variant.

    python tests/test_gpu_arith_edges.py sweep   runs the sweep on the library named by IBFT_LIB (one variant's subprocess)"""
import concurrent.futures
import os
import subprocess
import sys
import tempfile

import pytest

import arith_edges as AE

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = ["IBFT_KARATSUBA", "IBFT_REDUCE_SHIFT", "IBFT_SQR_VIA_MUL", "IBFT_PORTABLE_FE"]


def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def runner(e):
    return lambda op, a, b, stride: e.debug_op(op, a, b, out_stride=stride)


@pytest.fixture(scope="module")
def dev():
    _need_gpu()
    import ibft_b200 as ib
    e = ib.Engine(device=0)
    yield e
    e.close()


def test_arith_edge_sweep(dev):
    bad = AE.check_sweep(runner(dev))
    assert not bad, "\n".join(bad)


def test_chained_raw_sequences(dev):
    bad = AE.check_chains(runner(dev), lanes=256, steps=3000)
    assert not bad, "\n".join(bad)


@pytest.fixture(scope="session")
def variant_libs():
    """engine.cu built with the product's flags plus each variant's define, in parallel, into a temporary directory"""
    _need_gpu()
    import ibft_b200 as ib
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = tempfile.TemporaryDirectory(prefix="ibft_variants_")
    src = os.path.join(ib.build.CSRC, "engine.cu")

    def build(flag):
        so = os.path.join(tmp.name, f"lib_{flag}.so")
        p = subprocess.run([nvcc] + ib.build.NVCC_FLAGS + [f"-D{flag}", "-o", so, src], cwd=ib.build.CSRC, capture_output=True, text=True)
        return flag, so, p.returncode, p.stderr[-2000:]

    with concurrent.futures.ThreadPoolExecutor(len(VARIANTS)) as pool:
        built = {flag: (so, rc, err) for flag, so, rc, err in pool.map(build, VARIANTS)}
    yield built
    tmp.cleanup()


@pytest.mark.parametrize("flag", VARIANTS)
def test_variant_build_sweep(variant_libs, flag):
    """the field and scalar sweep against engine.cu built with -D<flag>, in a subprocess of its own"""
    so, rc, err = variant_libs[flag]
    assert rc == 0, f"-D{flag} does not build:\n{err}"
    env = dict(os.environ, IBFT_LIB=so, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests"), os.environ.get("PYTHONPATH", "")]))
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "sweep"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"-D{flag}: the sweep disagrees with the big-integer reference\n{p.stdout[-4000:]}{p.stderr[-4000:]}"


def _sweep_main():
    import ibft_b200 as ib
    e = ib.Engine(device=0)
    try:
        bad = AE.check_sweep(runner(e)) + AE.check_chains(runner(e), lanes=64, steps=500)
    finally:
        e.close()
    print("\n".join(bad) or "sweep ok")
    return 1 if bad else 0


if __name__ == "__main__" and sys.argv[1:] == ["sweep"]:
    sys.exit(_sweep_main())
