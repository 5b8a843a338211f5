"""The recover step's kernel choice (go-ibft_b200/csrc/recover_plan.hpp) against an independent model of the policy its header
comment states: AUTO's resolution, the kernels of every resolved path with and without the known-key pass, with and without a
combined generator table, and the cut of a host-buffer call into latency pieces -- at every threshold minus one, at it and plus
one, for 132 and 114 SMs."""
import ctypes
import itertools
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

AUTO, THREAD, QUAD, SPLIT, QSPLIT = 0, 1, 2, 3, 4   # IBFT_PATH_*
PATHS = (AUTO, THREAD, QUAD, SPLIT, QSPLIT)
# ibft::sig_kernel
KERNELS = {None: 0, "recover32": 1, "recover128": 2, "quad": 3, "split": 4, "qsplit": 5, "verify_known32": 6, "verify_known128": 7,
           "verify_split": 8}


@pytest.fixture(scope="module")
def rp(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "g++"))
    if cxx is None:
        pytest.fail("no C++ compiler to build the planner driver")
    so = str(tmp_path_factory.mktemp("recover_plan") / "librp.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "recover_plan_driver.cpp")])
    lib = ctypes.CDLL(so)
    I, U32 = ctypes.c_int, ctypes.c_uint32
    lib.rp_known.restype = I
    lib.rp_known.argtypes = [I, I, I, I, U32, U32]
    lib.rp_plan.restype = I
    lib.rp_plan.argtypes = [I, U32, ctypes.c_size_t, U32, I, I]
    lib.rp_pieces.restype = U32
    lib.rp_pieces.argtypes = [I, U32, ctypes.c_size_t, U32, I, I, ctypes.POINTER(I)]
    return lib


def model_plan(path, cnt, arena_len, sms, known, wc):
    """(first kernel, worklist kernel) of one recover step of cnt items"""
    small = cnt <= sms * 256
    long = arena_len // cnt > 256
    if path == AUTO:
        if not wc:
            path = QUAD if cnt <= sms * 32 else THREAD
        elif known or long:
            path = THREAD
        elif cnt <= sms * 48:
            path = QSPLIT
        elif cnt <= sms * 192:
            path = SPLIT
        else:
            path = THREAD
    thread = ("recover32" if small else "recover128", None)
    if not wc:
        return ("quad", None) if path == QUAD else thread
    if path == QSPLIT:
        return "qsplit", None
    if path == SPLIT:
        return ("verify_split", "qsplit") if known else ("split", None)
    if path == QUAD:
        return "quad", None
    if known:
        return "verify_known32" if small else "verify_known128", "qsplit" if small and not long else "recover128"
    return thread


def model_pieces(path, n, arena_len, sms, known, wc):
    """(items per piece, path of every piece); 0 items: the call goes in upload chunks on its own path"""
    if wc and path == AUTO and sms * 48 < n <= sms * 96 and arena_len // n <= 256:
        quarter = -(-n // 4)
        return -(-quarter // 96) * 96, THREAD if known else SPLIT
    return 0, path


def plan(rp, path, cnt, arena_len, sms, known, wc):
    v = rp.rp_plan(path, cnt, arena_len, sms, known, wc)
    return v // 16, v % 16


def edges(*points):
    return sorted({x + d for x in points for d in (-1, 0, 1) if x + d >= 1})


def arena_lengths(cnt):
    # around the long-payload cut: 256 bytes per item is not long, 256 + 1/cnt still is not (integer division), 257 is
    return (0, 256 * cnt - 1, 256 * cnt, 256 * cnt + cnt - 1, 257 * cnt, 1000 * cnt)


@pytest.mark.parametrize("sms", [132, 114])
def test_plan_matches_model(rp, sms):
    counts = edges(1, 24, 32, sms * 32, sms * 48, sms * 96, sms * 192, sms * 256, 1 << 17) + [1 << 20]
    checked = 0
    for cnt in counts:
        for arena_len, path, known, wc in itertools.product(arena_lengths(cnt), PATHS, (0, 1), (0, 1)):
            want = model_plan(path, cnt, arena_len, sms, known, wc)
            assert plan(rp, path, cnt, arena_len, sms, known, wc) == (KERNELS[want[0]], KERNELS[want[1]]), \
                (path, cnt, arena_len, sms, known, wc, want)
            checked += 1
    assert checked == len(counts) * 6 * len(PATHS) * 4


def test_auto_edges(rp):
    """AUTO at each size threshold, short payloads, without the known-key pass: the last count on a path and the first past it"""
    sms = 132
    for cnt, wc, want in [(sms * 48, 1, "qsplit"), (sms * 48 + 1, 1, "split"), (sms * 192, 1, "split"), (sms * 192 + 1, 1, "recover32"),
                          (sms * 256, 1, "recover32"), (sms * 256 + 1, 1, "recover128"), (sms * 32, 0, "quad"),
                          (sms * 32 + 1, 0, "recover32"), (sms * 256, 0, "recover32"), (sms * 256 + 1, 0, "recover128")]:
        assert plan(rp, AUTO, cnt, 100 * cnt, sms, 0, wc) == (KERNELS[want], 0), (cnt, wc)
    # long payloads and the key registry take the one-thread kernels whatever the size
    assert plan(rp, AUTO, 100, 257 * 100, sms, 0, 1) == (KERNELS["recover32"], 0)
    assert plan(rp, AUTO, 100, 0, sms, 1, 1) == (KERNELS["verify_known32"], KERNELS["qsplit"])
    assert plan(rp, AUTO, 100, 257 * 100, sms, 1, 1) == (KERNELS["verify_known32"], KERNELS["recover128"])


@pytest.mark.parametrize("sms", [132, 114])
def test_pieces_match_model(rp, sms):
    piece_path = ctypes.c_int()
    for n in [0] + edges(1, sms * 48, sms * 96, sms * 192):
        for arena_len, path, known, wc in itertools.product(arena_lengths(max(n, 1)), PATHS, (0, 1), (0, 1)):
            per = rp.rp_pieces(path, n, arena_len, sms, known, wc, ctypes.byref(piece_path))
            want = model_pieces(path, n, arena_len, sms, known, wc)
            assert (per, piece_path.value) == want, (path, n, arena_len, sms, known, wc)
            if per:
                # at most four pieces, each a whole number of k_recover_split CTAs; the last may be short or absent
                assert per % 96 == 0 and 4 * per >= n
                # each piece runs the kernels of its forced path: the known-key pass in one-warp CTAs, else chain + helper warps
                for lo in range(0, n, per):
                    cnt = min(per, n - lo)
                    first, second = plan(rp, piece_path.value, cnt, arena_len, sms, known, wc)
                    if known:
                        assert (first, second) == (KERNELS["verify_known32"], KERNELS["qsplit"] if arena_len // cnt <= 256 else
                                                   KERNELS["recover128"])
                    else:
                        assert (first, second) == (KERNELS["split"], 0)


def test_known_key_predicate(rp):
    for key_cache, want_recovered, groups, worklist in itertools.product((0, 1), repeat=4):
        for cap in (1, 100, 1 << 20):
            for cnt in (cap - 1, cap, cap + 1):
                want = key_cache and not want_recovered and groups and worklist and cnt <= cap
                assert rp.rp_known(key_cache, want_recovered, groups, worklist, cnt, cap) == int(bool(want))
