"""The out-of-place Jacobian's result kernels on the device: kernel time, byte model and the streaming ceiling of the same
read:write mix measured in the same run.

    python scripts/oop_bench.py [--reps R] [--out FILE]

Workloads (the native synthetic stencil fdbs_tridiag, forward mode, cyclic colours 1:3):
  sparse   the sparse result at C2 size: N = 10^7 tridiagonal sparsity and SparseMatrixCSC prototype, 3*10^7 candidate
           entries.  Kernel: oop_compact in its fused form (the quotient formed from the resident f outputs, then the
           zero-dropping compaction with the decoupled look-back).  Byte model: reads each entry's row (4 B) and colour
           (1 B), the f outputs once (8 B per row and colour, plus f(x)) and the column starts (4 B per column); writes
           rowval and nzval (16 B) per kept entry and colptr (8 B per column).  Ceiling: fdbs_stream_probe at 1:1 (the
           model is about 510:560 MB here, every quotient being nonzero).  Also reported: the whole sparse result, every
           library kernel of the call (step sizes, points, compaction, the look-back reset) without f's own kernels.
  dense    a dense result with a CSC sparsity at m = n = 3*10^4 (7.2 GB).  Kernels: the zero fill of J (cudaMemset), the
           existing explicit-destination scatter (diff_scatter_dest) and oop_plus_zero_slots (0.0 + q on the structural
           slots).  Byte model: 8mn written by the fill; the epilogue reads the destinations (8 B) and the slot (8 B) and
           writes the slot (8 B) per entry.  Ceilings: fdbs_store_probe (mode 0) for the fill, fdbs_stream_probe 2:1 for
           the epilogue's stream (it is a gather in the slots, so below it is expected).
Kernel times are per-kernel device durations from a torch.profiler trace of R calls, median over the calls.  Parity of
the sparse result with the CPU restatement is checked on the first 10^6 columns.  Prints one JSON line; the card's name,
power limit and maximum SM clock are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import torch  # noqa: E402

import _bootstrap  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def probe(pkg, n, mixes, reps):
    """GB/s of fdbs_stream_probe per (reads, writes) mix and of fdbs_store_probe ("store"): best over a few grids."""
    S = pkg._lib.synth()
    src = torch.empty(3 * n + 8, dtype=torch.float64, device="cuda").uniform_()
    dst = torch.empty(3 * n + 8, dtype=torch.float64, device="cuda")
    sink = torch.zeros(1, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {}
    for key in list(mixes) + ["store"]:
        best = 0.0
        for blocks in (sms * 4, sms * 8, sms * 16):
            if key == "store":
                run = lambda: S.fdbs_store_probe(dst.data_ptr(), 3 * n, 0, blocks, None)
                nbytes = 8.0 * 3 * n
            else:
                r, w = key
                run = lambda: S.fdbs_stream_probe(src.data_ptr(), n, r, dst.data_ptr(), n, w, n, blocks, sink.data_ptr(),
                                                  None)
                nbytes = 8.0 * n * (r + w)
            assert run() == 0
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            best = max(best, nbytes * reps / (e0.elapsed_time(e1) * 1e-3) / 1e9)
        out["store" if key == "store" else f"{key[0]}:{key[1]}"] = best
    return out


def kernel_times(fn, reps):
    """{kernel name: median device ms per call} from a torch.profiler trace of `reps` calls"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    per = {}
    for e in events:
        if e.get("cat") in ("kernel", "gpu_memset"):
            name = e["name"]
            short = next((k for k in ("oop_compact", "oop_plus_zero_slots", "diff_scatter_dest", "diff_scatter_staged",
                                      "diff_scatter_ident", "perturb_colors", "color_sumsq", "fdbs_tridiag")
                          if k in name), "memset" if e.get("cat") == "gpu_memset" else name[:40])
            per.setdefault(short, []).append(float(e["dur"]) / 1e3)
    return {k: float(np.median(v)) for k, v in per.items() if len(v) >= reps}, {k: len(v) for k, v in per.items()}


def tridiag(pkg, n):
    from _util import tridiag_csc
    cp, rv = tridiag_csc(n)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp).cuda(), torch.from_numpy(rv).cuda(),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    return S, cp, rv


def _row(ms, rbytes, wbytes, mix, ceil):
    gbs = (rbytes + wbytes) / (ms * 1e-3) / 1e9
    return {"ms": round(ms, 4), "read_bytes": int(rbytes), "write_bytes": int(wbytes), "GBps": round(gbs, 1),
            "mix": mix, "ceiling_GBps": round(ceil[mix], 1), "share_of_ceiling": round(gbs / ceil[mix], 3)}


def bench_sparse(pkg, n, reps, ceil):
    L = pkg._lib
    S, cp, rv = tridiag(pkg, n)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0x5EED + 2, None)
    ctx = L.TridiagCtx(n, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    cv = torch.from_numpy((np.arange(n) % 3 + 1).astype(np.int64)).cuda()
    cache = pkg.JacobianCache(x, "forward")
    call = lambda: pkg.finite_difference_jacobian(f, x, cache, sparsity=S, colorvec=cv, jac_prototype=S)
    J = call()
    for _ in range(3):
        call()
    t, counts = kernel_times(call, reps)
    E, nnz = len(rv), J.nnz
    # parity on the first 10^6 columns: the stencil's quotients with the device's step sizes
    import _literal_oop as LO
    k = 1_000_000
    xh = x.cpu().numpy()
    eps = list(cache._last_plan.eps())
    want = LO.jacobian_oop_csc_fast(orc_tridiag, xh, "forward", eps, n, cp, rv, cv.cpu().numpy())
    cut = int(want[3][k] - 1)
    parity = bool(np.array_equal(J.colptr[: k + 1].cpu().numpy(), want[3][: k + 1]) and
                  np.array_equal(J.rowval[:cut].cpu().numpy(), want[4][:cut]) and
                  np.array_equal(J.nzval[:cut].cpu().numpy().view(np.uint64), want[5][:cut].view(np.uint64)))
    return {"n": n, "candidates": E, "kept": nnz, "bit_identical_first_1e6_columns": parity,
            "oop_compact": _row(t["oop_compact"], 5 * E + 8 * n * 4 + 4 * (n + 1), 16 * nnz + 8 * (n + 1), "1:1", ceil),
            "sparse_result_library_ms": round(sum(v for k2, v in t.items() if "tridiag" not in k2), 4),
            "all_kernels_ms": {k2: round(v, 4) for k2, v in t.items()}, "launches_per_call": counts}


def orc_tridiag(v):
    """CPU twin of fdbs_tridiag: dx[i] = x[i-1] - 2x[i] + x[i+1] (test/coloring_tests.jl:5-13), in its order"""
    xm = np.concatenate([[0.0], v[:-1]])
    xp = np.concatenate([v[1:], [0.0]])
    return (xm - 2.0 * v) + xp


def bench_dense(pkg, n, reps, ceil):
    L = pkg._lib
    S, cp, rv = tridiag(pkg, n)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0x5EED + 3, None)
    ctx = L.TridiagCtx(n, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    cv = torch.from_numpy((np.arange(n) % 3 + 1).astype(np.int64)).cuda()
    cache = pkg.JacobianCache(x, "forward")
    out = {}

    def call():
        out["J"] = None
        out["J"] = pkg.finite_difference_jacobian(f, x, cache, sparsity=S, colorvec=cv)

    for _ in range(3):
        call()
    t, counts = kernel_times(call, reps)
    E = len(rv)
    res = {"m": n, "n": n, "J_bytes": 8 * n * n, "structural": E,
           "zero_fill": _row(t["memset"], 0, 8 * n * n, "store", ceil),
           "oop_plus_zero_slots": _row(t["oop_plus_zero_slots"], 16 * E, 8 * E, "2:1", ceil),
           "diff_scatter_dest_ms": round(t.get("diff_scatter_dest", float("nan")), 4),
           "all_kernels_ms": {k: round(v, 4) for k, v in t.items()}, "launches_per_call": counts}
    res["epilogue_share_of_result_time"] = round(t["oop_plus_zero_slots"] / (t["memset"] + t["oop_plus_zero_slots"] +
                                                                            t.get("diff_scatter_dest", 0.0)), 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n-sparse", type=int, default=10_000_000)
    ap.add_argument("--n-dense", type=int, default=30_000)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("oop_bench.py measures the device path and needs a GPU")
    pkg = _bootstrap.load_package()
    ceil = probe(pkg, 100_000_000, [(1, 1), (2, 1)], 20)
    res = {"card": card(), "probe_ceilings_GBps": {k: round(v, 1) for k, v in ceil.items()}}
    res["sparse_c2"] = bench_sparse(pkg, a.n_sparse, a.reps, ceil)
    torch.cuda.empty_cache()
    res["dense_csc"] = bench_dense(pkg, a.n_dense, a.reps, ceil)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
