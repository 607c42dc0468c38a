"""The banded out-of-place Jacobian (fdb_oop_plan_create_banded) against the CSC route on the CSC of the same band: plan
build, per-call time and kernel times, with the byte model of each result kernel and the streaming ceiling measured in
the same run.

    python scripts/oop_banded_bench.py [--reps R] [--out FILE]

Workloads (the native synthetic stencil fdbs_tridiag, cyclic colours):
  plan     N = 10^7, l = u = 1, 3 colours, sparse result: the band plan's build against the CSC route's, the latter
           including building the CSC of the band on the host (3*10^7 row indices).
  sparse   the same problem, forward and central: host time per call (ending in the result's one synchronisation) and
           the median device time per kernel from a separate torch.profiler run.  The band compaction (oop_compact in
           band form, fused) reads the f outputs once (8 B per row and colour, plus f(x) forward / the minus outputs
           central) and no row, colour or column-start stream; it writes rowval and nzval (16 B) per kept entry and colptr
           (8 B per column).  The CSC route's fused pass also reads the row (4 B) and colour (1 B) of every entry and the
           column starts (4 B per column).  Ceiling: fdbs_stream_probe at 1:1.
  dense    a dense result of the band at m = n = 3*10^4: zero fill, band scatter into the dense target, and the
           closed-form + 0.0 pass (oop_band_plus_zero: 8 B read and written per entry; ceiling fdbs_stream_probe 1:1).
  wide     l = u = 64, n = 10^6, 129 colours, sparse result with a scratch budget that splits the colours into several
           groups: the band scatter writes band data and the compaction copies from it (kCopy: 8 B read per entry).
Every band result is compared bit for bit with the CSC route's.  Prints one JSON line; the card's name, power limit and
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
from oop_bench import _row, card, kernel_times, probe  # noqa: E402


def band_csc_host(n, l, u):
    """CSC of the square band (l, u), 1-based, built on the host as a mirror user converting a band would"""
    c = np.arange(n, dtype=np.int64)
    lo, hi = np.maximum(c - u, 0), np.minimum(c + l, n - 1)
    cnt = hi - lo + 1
    colptr = np.concatenate([[1], 1 + np.cumsum(cnt)]).astype(np.int64)
    starts = np.repeat(colptr[:-1] - 1, cnt)
    rowval = np.repeat(lo, cnt) + (np.arange(int(cnt.sum()), dtype=np.int64) - starts) + 1
    return colptr, rowval


def problem(pkg, n, seed):
    L = pkg._lib
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), n, seed, None)
    ctx = L.TridiagCtx(n, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    return x, f


def proto(pkg, n):
    return pkg.SparseMatrixCSC(n, n, torch.ones(n + 1, dtype=torch.int64), torch.zeros(0, dtype=torch.int64), None)


def same(a, b):
    if isinstance(a, torch.Tensor):
        return bool(torch.equal(a.view(torch.int64), b.view(torch.int64)))
    return bool(torch.equal(a.colptr, b.colptr) and torch.equal(a.rowval, b.rowval) and
                torch.equal(a.nzval.view(torch.int64), b.nzval.view(torch.int64)))


def timed(call, reps):
    call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        call()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def bench_plan_and_sparse(pkg, n, reps, ceil):
    L = pkg._lib
    cv = torch.from_numpy((np.arange(n) % 3 + 1).astype(np.int64)).cuda()
    x, f = problem(pkg, n, 0x5EED + 2)
    res = {"n": n, "l": 1, "u": 1, "colours": 3}
    B = pkg.BandedMatrix(n, n, 1, 1)
    for fd in ("forward", "central"):
        caches = {k: pkg.JacobianCache(x, fd) for k in ("band", "csc")}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        caches["band"]._oop_plan_for(L.FDB_OOP_SPARSE, B, cv, n, n, n, x.device)
        torch.cuda.synchronize()
        t_band = time.perf_counter() - t0
        t0 = time.perf_counter()
        cp, rv = band_csc_host(n, 1, 1)
        S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), None)
        caches["csc"]._oop_plan_for(L.FDB_OOP_SPARSE, S, cv, n, n, n, x.device)
        torch.cuda.synchronize()
        t_csc = time.perf_counter() - t0
        if fd == "forward":
            res["plan_build_s"] = {"band": round(t_band, 4), "csc_with_host_csc": round(t_csc, 4)}
        sps = {"band": B, "csc": S}
        calls = {k: (lambda k=k: pkg.finite_difference_jacobian(f, x, caches[k], sparsity=sps[k], colorvec=cv,
                                                                 jac_prototype=proto(pkg, n))) for k in sps}
        out = {"bit_identical": same(calls["band"](), calls["csc"]())}
        for k in ("band", "csc", "band", "csc"):   # alternated, the second round kept
            out[f"{k}_call_ms"] = round(timed(calls[k], reps), 4)
        kept = int(calls["band"]().nnz)
        slabs = 3 * 8 * n * (2 if fd == "central" else 1) + (8 * n if fd == "forward" else 0)
        wbytes = 16 * kept + 8 * (n + 1)
        E = 3 * n - 2
        for k in ("band", "csc"):
            t, counts = kernel_times(calls[k], reps)
            rbytes = slabs + (0 if k == "band" else 5 * E + 4 * (n + 1))
            out[f"{k}_oop_compact"] = _row(t["oop_compact"], rbytes, wbytes, "1:1", ceil)
            out[f"{k}_kernels_ms"] = {k2: round(v, 4) for k2, v in t.items()}
        res[f"sparse_{fd}"] = out
    return res


def bench_dense(pkg, n, reps, ceil):
    cv = torch.from_numpy((np.arange(n) % 3 + 1).astype(np.int64)).cuda()
    x, f = problem(pkg, n, 0x5EED + 3)
    B = pkg.BandedMatrix(n, n, 1, 1)
    cache = pkg.JacobianCache(x, "forward")
    out = {}

    def call():
        out["J"] = None
        out["J"] = pkg.finite_difference_jacobian(f, x, cache, sparsity=B, colorvec=cv)

    call()
    ms = timed(call, reps)
    t, _ = kernel_times(call, reps)
    t = {("oop_band_plus_zero" if "oop_band_plus_zero" in k else k): v for k, v in t.items()}
    E = 3 * n - 2
    band_j = out["J"].clone()
    out["J"] = None
    cp, rv = band_csc_host(n, 1, 1)
    csc_j = pkg.finite_difference_jacobian(f, x, pkg.JacobianCache(x, "forward"), colorvec=cv,
                                           sparsity=pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), None))
    ident = same(band_j, csc_j)
    del band_j, csc_j
    return {"m": n, "n": n, "J_bytes": 8 * n * n, "bit_identical": ident, "call_ms": round(ms, 4),
            "zero_fill": _row(t["memset"], 0, 8 * n * n, "store", ceil),
            "oop_band_plus_zero": _row(t["oop_band_plus_zero"], 8 * E, 8 * E, "1:1", ceil),
            "kernels_ms": {k: round(v, 4) for k, v in t.items()}}


def bench_wide(pkg, n, reps, ceil):
    L = pkg._lib
    l = u = 64
    C_ = l + u + 1
    cv = torch.from_numpy((np.arange(n) % C_ + 1).astype(np.int64)).cuda()
    x, f = problem(pkg, n, 0x5EED + 4)
    B = pkg.BandedMatrix(n, n, l, u)
    cache = pkg.JacobianCache(x, "forward", scratch_bytes=256 << 20)
    call = lambda: pkg.finite_difference_jacobian(f, x, cache, sparsity=B, colorvec=cv, jac_prototype=proto(pkg, n))
    J = call()
    info = cache._last_plan.info()
    cp, rv = band_csc_host(n, l, u)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), None)
    Jc = pkg.finite_difference_jacobian(f, x, pkg.JacobianCache(x, "forward", scratch_bytes=256 << 20), sparsity=S,
                                        colorvec=cv, jac_prototype=proto(pkg, n))
    ident = same(J, Jc)
    del Jc
    ms = timed(call, reps)
    t, _ = kernel_times(call, reps)
    E, kept = info["n_entries"], int(J.nnz)
    return {"n": n, "l": l, "u": u, "colours": C_, "groups": info["n_groups"], "candidates": E, "bit_identical": ident,
            "call_ms": round(ms, 4),
            "oop_compact_copy": _row(t["oop_compact"], 8 * E, 16 * kept + 8 * (n + 1), "1:1", ceil),
            "kernels_ms": {k: round(v, 4) for k, v in t.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--n-dense", type=int, default=30_000)
    ap.add_argument("--n-wide", type=int, default=1_000_000)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("oop_banded_bench.py measures the device path and needs a GPU")
    pkg = _bootstrap.load_package()
    ceil = probe(pkg, 100_000_000, [(1, 1)], 20)
    res = {"card": card(), "probe_ceilings_GBps": {k: round(v, 1) for k, v in ceil.items()}}
    res["c2"] = bench_plan_and_sparse(pkg, a.n, a.reps, ceil)
    torch.cuda.empty_cache()
    res["dense"] = bench_dense(pkg, a.n_dense, a.reps, ceil)
    torch.cuda.empty_cache()
    res["wide"] = bench_wide(pkg, a.n_wide, a.reps, ceil)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
