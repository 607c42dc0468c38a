"""The block out-of-place Jacobians (fdb_oop_plan_create_block_banded / _block_dense) against the CSC route on the CSC of
the same entry set: plan build, per-call time and the compaction kernel's time, with its byte model over the streaming
ceiling measured in the same run.

    python scripts/oop_block_bench.py [--reps R] [--out FILE]

Workloads (sparse result, f the native synthetic fdbs_tridiag, matrix_colors):
  stencil  the 5-point structure of a g x g grid, g = 1000: a BandedBlockBandedMatrix of 1000 blocks of 1000 with
           (l, u) = (1, 1) and (lam, mu) = (1, 1), 9 colours, 8.988*10^6 entries.
  blocks8  a BlockSkylineMatrix of 2.5*10^5 blocks of 8 with (l, u) = (1, 1): n = 2*10^6, 24 colours, 4.8*10^7 entries.
Each in forward and central mode:
  plan_build_s   the block plan's build against the CSC route's, the latter including building the CSC of E on the host
                 (the mirror's findstructralnz, sorted into CSC order) as a caller converting the structure would;
  call_ms        host time per whole mirror call (ending in the result's one synchronisation), routes alternated;
  oop_compact    the median device time of the compaction from a separate torch.profiler run.  The block compaction
                 reads the f outputs once per entry (8 B, plus f(x) forward or the minus outputs central) and no row,
                 colour or column-start stream; it writes rowval and nzval (16 B) per kept entry and colptr (8 B per
                 column).  The CSC route's fused pass also reads each entry's row (4 B) and colour (1 B) and the column
                 starts (4 B per column).  Ceiling: fdbs_stream_probe at 1:1.
Every block result is compared bit for bit with the CSC route's.  Prints one JSON line; the card's name, power limit and
maximum SM clock are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "scripts"))

import torch  # noqa: E402

import _bootstrap  # noqa: E402
from oop_banded_bench import problem, proto, same, timed  # noqa: E402
from oop_bench import _row, card, kernel_times, probe  # noqa: E402


def host_csc(sp):
    """CSC of the structure's entry set, 1-based, from findstructralnz on the host"""
    r, c, _ = sp.findstructralnz()
    o = np.lexsort((r, c))
    r, c = r[o], c[o]
    colptr = np.concatenate([[1], 1 + np.cumsum(np.bincount(c - 1, minlength=sp.shape[1]))]).astype(np.int64)
    return colptr, r.astype(np.int64)


def bench(pkg, name, sp, reps, ceil):
    L = pkg._lib
    n = sp.shape[1]
    cv = torch.from_numpy(sp.matrix_colors()).cuda()
    Cn = int(cv.max())
    x, f = problem(pkg, n, 0x5EED + 7)
    res = {"n": n, "colours": Cn}
    for fd in ("forward", "central"):
        caches = {k: pkg.JacobianCache(x, fd) for k in ("block", "csc")}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        caches["block"]._oop_plan_for(L.FDB_OOP_SPARSE, sp, cv, n, n, n, x.device)
        torch.cuda.synchronize()
        t_block = time.perf_counter() - t0
        t0 = time.perf_counter()
        cp, rv = host_csc(sp)
        S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), None)
        caches["csc"]._oop_plan_for(L.FDB_OOP_SPARSE, S, cv, n, n, n, x.device)
        torch.cuda.synchronize()
        t_csc = time.perf_counter() - t0
        E = len(rv)
        res["entries"] = E
        if fd == "forward":
            res["plan_build_s"] = {"block": round(t_block, 4), "csc_with_host_csc": round(t_csc, 4)}
        sps = {"block": sp, "csc": S}
        calls = {k: (lambda k=k: pkg.finite_difference_jacobian(f, x, caches[k], sparsity=sps[k], colorvec=cv,
                                                                 jac_prototype=proto(pkg, n))) for k in sps}
        out = {"bit_identical": same(calls["block"](), calls["csc"]())}
        for k in ("block", "csc", "block", "csc"):   # alternated, the second round kept
            out[f"{k}_call_ms"] = round(timed(calls[k], reps), 4)
        kept = int(calls["block"]().nnz)
        # each entry reads its colour's output (and f(x) forward / the minus output central) once
        reads = 8 * E * (2 if fd == "central" else 1) + (8 * E if fd == "forward" else 0)
        wbytes = 16 * kept + 8 * (n + 1)
        for k in ("block", "csc"):
            t, _ = kernel_times(calls[k], reps)
            if "oop_compact" not in t:                 # a profile that lost events: take it again
                t, _ = kernel_times(calls[k], reps)
            rbytes = reads + (0 if k == "block" else 5 * E + 4 * (n + 1))
            out[f"{k}_oop_compact"] = _row(t["oop_compact"], rbytes, wbytes, "1:1", ceil)
            out[f"{k}_kernels_ms"] = {k2: round(v, 4) for k2, v in t.items()}
        res[fd] = out
        del caches, calls, S
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--g", type=int, default=1000)
    ap.add_argument("--blocks", type=int, default=250_000)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("oop_block_bench.py measures the device path and needs a GPU")
    pkg = _bootstrap.load_package()
    ceil = probe(pkg, 100_000_000, [(1, 1)], 20)
    res = {"card": card(), "probe_ceilings_GBps": {k: round(v, 1) for k, v in ceil.items()}}
    res["stencil"] = bench(pkg, "stencil", pkg.BandedBlockBandedMatrix([a.g] * a.g, [a.g] * a.g, (1, 1), (1, 1)),
                           a.reps, ceil)
    res["blocks8"] = bench(pkg, "blocks8", pkg.BlockSkylineMatrix([8] * a.blocks, [8] * a.blocks, (1, 1)), a.reps, ceil)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
