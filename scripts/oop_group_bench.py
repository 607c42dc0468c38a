"""Multi-GPU out-of-place Jacobians (fdb_group_jacobian_oop): time per call of the single plan and of groups over repeated
and distinct devices, with every group's result bit-compared with the single plan's.

    python scripts/oop_group_bench.py [--out FILE]

Two sparse results (SparseMatrixCSC prototype = the sparsity), forward mode, native synthetic f:
  c4   N = 5*10^6, the random 8-entries-per-row f of bench.py's C4 (fdbs_ellrows, the same instance), 64 cyclic colours:
       f dominates the call;
  c2   N = 10^7 tridiagonal (fdbs_tridiag), 3 cyclic colours: the result kernels dominate.
Arms: the single plan (finite_difference_jacobian with a JacobianCache); group [0]; group [0, 0] (two members on one
card: stream overlap and the group's overhead, not scaling); and, when k > 1 GPUs are visible, group [0 .. k-1].  A call
is the whole mirror call: f(x), the colours, the compaction and the one host sync that sizes the result.  Each arm is
warmed up, then timed with CUDA events on the root stream over more than one second of calls, in three rounds that
alternate the arms; call_s is the best round, spread the (max - min) / min of the rounds.  The root's compaction
(oop_compact) is timed per call from a torch.profiler trace of its own, after the timed rounds.  Prints one JSON line;
the card's name, power limit and max SM clock are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import _bootstrap  # noqa: E402
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


class Problem:
    """x, the CSC sparsity (also the prototype), the colours and one native f per device"""

    def __init__(self, pkg, workload):
        self.pkg, self.workload = pkg, workload
        dev = torch.device("cuda", 0)
        L = pkg._lib
        if workload == "c4":
            n, K, Cc = bench.C4_N, bench.C4_K, bench.C4_C
            self.cols, self.coef = bench.c4_instance_torch(dev, n, K, Cc)
            cols64 = self.cols.to(torch.int64)
            rows = torch.arange(n, device=dev, dtype=torch.int64).repeat(K)
            order = torch.argsort(cols64.reshape(-1) * n + rows)
            rowval = (rows[order] + 1).contiguous()
            colptr = torch.cat([torch.ones(1, dtype=torch.int64, device=dev),
                                1 + torch.cumsum(torch.bincount(cols64.reshape(-1), minlength=n), 0)])
            del cols64, rows, order
            self.K, seed = K, bench.SEED + 4
        else:
            n, Cc = 10_000_000, 3
            colptr, rowval = bench.tridiag_pattern_torch(n, dev)
            seed = bench.SEED + 2
        self.n, self.C = n, Cc
        self.cv = (torch.arange(n, dtype=torch.int64, device=dev) % Cc) + 1
        self.x = torch.empty(n, dtype=torch.float64, device=dev)
        L.synth().fdbs_fill_x(self.x.data_ptr(), n, seed, None)
        self.S = pkg.SparseMatrixCSC(n, n, colptr, rowval, torch.zeros(rowval.numel(), dtype=torch.float64, device=dev))
        self._keep = []

    def fn(self, d):
        L = self.pkg._lib
        if self.workload == "c4":
            dev = torch.device("cuda", d)
            cols, coef = self.cols.to(dev), self.coef.to(dev)
            ctx = L.EllCtx(self.n, self.K, cols.data_ptr(), coef.data_ptr(), 0)
            self._keep.append((cols, coef, ctx))
            return self.pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx)
        ctx = L.TridiagCtx(self.n, 0)
        self._keep.append(ctx)
        return self.pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)


def timed(call, min_s=1.0):
    """seconds per call: one warm-up call, one call to size the window, then >= min_s of calls between two events on the
    current (root) stream"""
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    torch.cuda.synchronize()
    reps = max(3, math.ceil(1.2 * min_s / (e0.elapsed_time(e1) / 1e3)))
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def compaction_ms(call, reps=5):
    """median device time of oop_compact per call, from a torch.profiler trace of `reps` calls"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    ms = [float(e["dur"]) / 1e3 for e in events if e.get("cat") == "kernel" and "oop_compact" in e["name"]]
    return float(np.median(ms)) if ms else None


def same_bits(a, b):
    return (a.m, a.n) == (b.m, b.n) and torch.equal(a.colptr, b.colptr) and torch.equal(a.rowval, b.rowval) and \
        torch.equal(a.nzval.view(torch.int64), b.nzval.view(torch.int64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "oop_group_bench needs a GPU"
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import distributed
    k = torch.cuda.device_count()
    res = {"metric": "oop_group_jacobian", "card": card(), "visible_gpus": k, "fdtype": "forward", "result": "sparse"}
    arms = [[0], [0, 0]] + ([list(range(k))] if k > 1 else [])
    rounds = 3
    res["rounds"] = rounds
    for workload in ("c4", "c2"):
        p = Problem(pkg, workload)
        cache = pkg.JacobianCache(p.x, "forward")
        f0 = p.fn(0)
        out = {}

        def single():
            out["single"] = pkg.finite_difference_jacobian(f0, p.x, cache, sparsity=p.S, colorvec=p.cv, jac_prototype=p.S)

        calls, groups = {"single": single}, {}
        for devices in arms:
            name = "group_" + "_".join(map(str, devices))
            g = distributed.GroupJacobianOOP(devices, "forward", colorvec=p.cv, sparsity=p.S, jac_prototype=p.S)
            fs = [p.fn(d) for d in devices]
            groups[name] = g

            def call(g=g, fs=fs, name=name):
                out[name] = g.run(fs, p.x)
            calls[name] = call
        # the arms alternate round by round, so that clock and neighbour drift fall on all of them alike
        times = {name: [] for name in calls}
        for _ in range(rounds):
            for name, call in calls.items():
                times[name].append(timed(call))
        best = {name: min(v) for name, v in times.items()}
        row = {"n": p.n, "colors": p.C, "candidates": int(p.S.rowval.numel()), "kept": int(out["single"].nnz),
               "single": {"call_s": best["single"], "rounds_s": times["single"],
                          "spread": max(times["single"]) / min(times["single"]) - 1,
                          "compaction_ms": compaction_ms(single)}}
        for name, g in groups.items():
            row[name] = {
                "call_s": best[name], "rounds_s": times[name], "spread": max(times[name]) / min(times[name]) - 1,
                "speedup_vs_single": best["single"] / best[name],
                "member_fcalls": [pl.info()["fcalls_per_jacobian"] for pl in g.plans],
                "root_compaction_ms": compaction_ms(calls[name]),
                "bit_identical_to_single": bool(same_bits(out[name], out["single"]))}
            g.close()
        res[workload] = row
        del p, cache, out, calls, groups
        torch.cuda.empty_cache()
    res["scaling"] = "measured" if k > 1 else "not measured: one GPU visible ([0, 0] measures stream overlap and overhead)"
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
