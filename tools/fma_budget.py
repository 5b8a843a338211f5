#!/usr/bin/env python3
"""FMA-pipe ledger of the throughput recover kernel (k_recover<128>), computed on the CPU.

The recover kernel is bound by the FMA-heavy pipe (DESIGN.md §3.1): an IMAD.WIDE(.X) holds it for 4 cycles per warp
instruction, every other IMAD-class instruction (IMAD.MOV, IMAD.X, IMAD.HI, ...) for 2.  This tool puts a number on that
pipe's work per recovery without a GPU:

  static   the SASS of k_recover<128> (cuobjdump): every out-of-line routine it calls (fe_mul, fe_sqr, fe_sqrn, the doubling's
           fused front end, the safegcd inversion, the root-and-inverse exponentiation fe_sqrt_inv), the window loop and the
           u1*G comb loop after it, found by their back branches;
  dynamic  how often each of them runs per recovery, counted by the host emulation of the same sources (IBFT_OPCOUNT,
           tests/emul/recover_comb.cpp: the product's one-thread composition) over the config-3 items (tests/golden/config3.npz).

It prints per-routine instruction counts, then estimated FMA-pipe cycles, IMAD.WIDE and products per recovery and the
hot-loop code size (window loop + every routine it calls outside the P + P block).  The estimate covers the field routines, the inversions and the
window loop and the comb loop.  The addition body is charged whole to every addition except its P + P block (listed apart,
never taken by the config-3 items); its other short branches (beta, negation, zero digits) are counted as taken, so that term
is an upper bound.  Keccak, range checks and the inline code of the final addition (its products are calls, counted above) are
not modelled.

  python tools/fma_budget.py                 # builds go-ibft_b200/libibftverify.so if stale
  IBFT_LIB=/path/libibftverify.so python tools/fma_budget.py --items 2000
"""
from __future__ import annotations

import argparse
import ctypes
import importlib.util
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_Z9k_recoverILi128EEvPK13ibft_sig_itemjPKhmjjPK15ibft_group_descjPK8slot_devjPjPhSC_PKj9vote_sinkSE_"
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")

# IBFT_OP_* of csrc/secp_fe.cuh
OPS = ["mul_body", "sqr_body", "mul_call", "sqr_call", "sqrn_call", "sqrn_iter", "dbl_front", "fe_inv", "sc_inv", "inv_iter",
       "win", "win_dbl", "win_add", "comb_add", "rec_final"]
# demangled-name fragment of an out-of-line routine -> its call counter
ROUTINES = [("fe_mul", "mul_call"), ("fe_sqrn", "sqrn_call"), ("fe_sqr", "sqr_call"), ("jac_dbl_front", "dbl_front"),
            ("fe_inv_safegcd", "fe_inv"), ("sc_inv_safegcd", "sc_inv"), ("fe_sqrt_inv", "rec_final")]
# routines with an inner loop: the counter of that loop's iterations
LOOPS = {"fe_sqrn": "sqrn_iter", "fe_inv_safegcd": "inv_iter", "sc_inv_safegcd": "inv_iter"}


def library() -> str:
    lib = os.environ.get("IBFT_LIB")
    if lib:
        return lib
    spec = importlib.util.spec_from_file_location("ibft_build", os.path.join(ROOT, "go-ibft_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()


def parse_sass(text: str):
    out = []
    for line in text.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            out.append((int(m.group(1), 16), m.group(2)))
    return out


def kernel_sass(lib: str):
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", KERNEL, lib], capture_output=True, text=True, check=True).stdout
    sym = subprocess.run([CUOBJDUMP, "-elf", lib], capture_output=True, text=True, check=True).stdout
    routines = {}
    for line in sym.splitlines():
        # local symbols of the routines ptxas placed in the kernel's section: "$<kernel>$<routine>"  value  size
        m = re.match(r"\s*0x[0-9a-f]+\s+0x([0-9a-f]+)\s+0x([0-9a-f]+)\s.*\$" + re.escape(KERNEL) + r"\$(\S+)", line)
        if m:
            routines[m.group(3)] = (int(m.group(1), 16), int(m.group(2), 16))
    return parse_sass(sass), routines


def opcode(ins: str) -> str:
    t = ins.split()
    if t[0].startswith("@"):
        t = t[1:]
    return t[0] if t else ""


def tally(ins):
    c = {"wide": 0, "imad": 0, "mov": 0, "hi": 0, "call": 0, "n": len(ins)}
    for _, t in ins:
        op = opcode(t)
        if op.startswith("IMAD.WIDE"):
            c["wide"] += 1
        elif op.startswith("IMAD"):
            c["imad"] += 1
            c["mov"] += op.startswith("IMAD.MOV")
            c["hi"] += op.startswith("IMAD.HI")
        elif op.startswith("CALL"):
            c["call"] += 1
    c["fma"] = 4 * c["wide"] + 2 * c["imad"]
    return c


def loops(ins):
    """(head, tail) of every back branch"""
    out = []
    for a, t in ins:
        m = re.search(r"\bBRA\b.*0x([0-9a-f]+)$", t)
        if m and int(m.group(1), 16) < a:
            out.append((int(m.group(1), 16), a))
    return out


def span(ins, lo, hi):
    return [x for x in ins if lo <= x[0] <= hi]


def window_loop(body):
    """the window loop: the loop holding the most nested loops that make calls; its first two such loops are the doubling
    loop and the loop over the digit streams (source order)"""
    lps = [(h, t) for h, t in loops(body) if tally(span(body, h, t))["call"]]
    best = None
    for h, t in lps:
        inner = sorted((h2, t2) for h2, t2 in lps if h <= h2 and t2 <= t and (h2, t2) != (h, t))
        if len(inner) >= 2 and (best is None or (len(inner), t - h) > (len(best[1]), best[0][1] - best[0][0])):
            best = ((h, t), inner)
    if best is None:
        raise SystemExit("window loop not found in the SASS")
    (h, t), inner = best
    # keep the outermost inner loops only
    top = [x for x in inner if not any(y != x and y[0] <= x[0] and x[1] <= y[1] for y in inner)]
    return (h, t), top[0], top[1]


def cold_block(add_loop, bounds, names):
    """the P + P branch of the mixed addition (a doubling, taken only by crafted signatures): the smallest region that a
    conditional forward branch jumps over, ends in an unconditional branch and holds either a whole inlined doubling (three
    calls or more) or the call of the out-of-line one"""
    def doubling(reg):
        calls = [x for x in reg if opcode(x[1]).startswith("CALL")]
        return len(calls) >= 3 or any("jac_double" in names.get(int(x[1].split()[-1], 16), "") for x in calls)

    best = None
    for a, t in add_loop:
        m = re.match(r"@!?P\d+ BRA (?:!?P\d+, )?0x([0-9a-f]+)$", t)
        if not m or not a < int(m.group(1), 16) <= bounds[1]:
            continue
        tg = int(m.group(1), 16)
        reg = [x for x in add_loop if a < x[0] < tg]
        if reg and doubling(reg) and re.match(r"BRA 0x", reg[-1][1]):
            if best is None or len(reg) < len(best):
                best = reg
    return best or []


def comb_loop(body, window_tail):
    """the u1*G comb loop: the first loop after the window loop that makes calls (the prefetch loop before it makes none)"""
    after = sorted((h, t) for h, t in loops(body) if h > window_tail and tally(span(body, h, t))["call"])
    if not after:
        raise SystemExit("comb loop not found in the SASS")
    return after[0]


def counting_emulation(out_dir: str) -> ctypes.CDLL:
    """the host emulation of the product's one-thread composition with its operation counters (tests/emul/recover_comb.cpp)"""
    emul = os.path.join(ROOT, "tests", "emul")
    so = os.path.join(out_dir, "libibft_recover_comb.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", '-DEMUL_DIR="%s"' % emul, "-shared", "-o",
                           so, os.path.join(emul, "recover_comb.cpp"), "-lpthread"])
    return ctypes.CDLL(so)


def op_counts(items_limit: int):
    with tempfile.TemporaryDirectory() as tmp:
        E = counting_emulation(tmp)  # stays mapped after the directory is removed
    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"])
    arena = np.ascontiguousarray(d["arena"])
    if items_limit:
        items = items[:items_limit]
    out = (ctypes.c_uint8 * 20)()
    ap = arena.ctypes.data_as(ctypes.c_void_p)
    E.emul_verify_item_comb(items[0].ctypes.data_as(ctypes.c_void_p), ap, ctypes.c_size_t(len(arena)), out)  # builds the emulation's tables
    E.emul_op_reset()
    for i in range(len(items)):
        E.emul_verify_item_comb(items[i].ctypes.data_as(ctypes.c_void_p), ap, ctypes.c_size_t(len(arena)), out)
    buf = (ctypes.c_ulonglong * 32)()
    n = E.emul_op_counts_all(buf)
    assert n <= len(OPS), "IBFT_OP_* of secp_fe.cuh and OPS of this tool disagree"
    return {k: (buf[i] if i < n else 0) for i, k in enumerate(OPS)}, len(items)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--items", type=int, default=0, help="config-3 items to emulate (0 = all 20,000)")
    args = ap.parse_args()
    lib = library()
    ins, syms = kernel_sass(lib)
    first_routine = min(off for off, _ in syms.values()) if syms else ins[-1][0] + 16
    body = [x for x in ins if x[0] < first_routine]

    counts, n_items = op_counts(args.items)
    recoveries = counts["win"] / 33.0  # IBFT_NWIN_R windows per double-scalar multiplication
    if not recoveries:
        raise SystemExit("no recovery reached the window loop")
    per = {k: v / recoveries for k, v in counts.items()}

    rows = []  # (name, tally, executions per recovery)
    for sym, (off, size) in sorted(syms.items(), key=lambda kv: kv[1][0]):
        name, key = next(((n, k) for n, k in ROUTINES if re.search(r"\d" + n + r"E", sym)), (sym, None))
        r = span(ins, off, off + size - 1)
        if name in LOOPS:
            lp = loops(r)
            lh, lt = max(lp, key=lambda x: x[1] - x[0])
            inside = span(r, lh, lt)
            rows.append((name + " (per call)", tally([x for x in r if not lh <= x[0] <= lt]), per.get(key, 0.0)))
            share = per[LOOPS[name]] * (per.get(key, 0.0) / max(1e-9, per["fe_inv"] + per["sc_inv"])) if LOOPS[name] == "inv_iter" \
                else per[LOOPS[name]]
            rows.append((name + " (per iteration)", tally(inside), share))
        else:
            rows.append((name, tally(r), per.get(key, 0.0) if key else 0.0))

    (wh, wt), dl, sl = window_loop(body)
    wl = span(body, wh, wt)
    dbl_loop, add_loop = span(body, *dl), span(body, *sl)
    rest = [x for x in wl if not (dl[0] <= x[0] <= dl[1] or sl[0] <= x[0] <= sl[1])]
    cold = cold_block(add_loop, sl, {off: name for name, (off, _) in syms.items()})
    rows.append(("window loop: per window", tally(rest), per["win"]))
    rows.append(("window loop: doubling", tally(dbl_loop), per["win_dbl"]))
    rows.append(("window loop: stream/addition", tally([x for x in add_loop if x not in cold]), per["win_add"]))
    rows.append(("window loop: P + P block (rare)", tally(cold), 0.0))
    ch, ct = comb_loop(body, wt)
    rows.append(("comb loop: per addition", tally(span(body, ch, ct)), per["comb_add"]))

    print(f"library: {lib}")
    print(f"dynamic counts: host emulation of {n_items} config-3 items, {recoveries:.0f} double-scalar multiplications")
    print()
    print(f"{'routine':34s} {'IMAD.WIDE':>9s} {'other IMAD':>10s} {'IMAD.MOV':>8s} {'IMAD.HI':>7s} {'CALL':>5s} {'instr':>6s} "
          f"{'FMA cyc':>8s} {'runs/rec':>9s}")
    tot_fma = tot_wide = tot_hi = tot_mov = 0.0
    for name, c, k in rows:
        print(f"{name:34s} {c['wide']:9d} {c['imad']:10d} {c['mov']:8d} {c['hi']:7d} {c['call']:5d} {c['n']:6d} {c['fma']:8d} {k:9.1f}")
        tot_fma += c["fma"] * k
        tot_wide += c["wide"] * k
        tot_hi += c["hi"] * k
        tot_mov += c["mov"] * k
    print()
    print("per recovery (dynamic counts):")
    for k in OPS:
        print(f"  {k:12s} {per[k]:10.1f}")
    # hot loop: the window loop (its P + P block included) plus every routine called from it outside the P + P block
    called = {int(re.search(r"0x([0-9a-f]+)", t).group(1), 16) for x in wl if x not in cold and opcode(x[1]).startswith("CALL")
              for t in [x[1]]}
    hot = len(wl) + sum(len(span(ins, off, off + size - 1)) for off, size in syms.values() if off in called)
    print()
    print(f"products per recovery            {per['mul_body'] + per['sqr_body']:10.1f}  "
          f"({per['mul_body']:.1f} multiplications + {per['sqr_body']:.1f} squarings)")
    # ptxas sometimes splits a 32x32->64 product into IMAD (low half) + IMAD.HI: the same 4 pipe cycles as one IMAD.WIDE
    print(f"IMAD.WIDE per recovery           {tot_wide:10.0f}  (+ {tot_hi:.0f} IMAD.HI: split products and high halves)")
    print(f"IMAD.MOV per recovery            {tot_mov:10.0f}")
    print(f"FMA-pipe cycles per recovery     {tot_fma:10.0f}  (per warp of 32 recoveries; estimate)")
    print(f"hot-loop code                    {hot * 16:10d} B  ({hot} instructions: window loop {len(wl)} + "
          f"{len(called)} routines it calls)")


if __name__ == "__main__":
    sys.exit(main())
