"""Diagonal-storage Jacobians: the banded plan with FDB_J_DIAGONALS (closed-form diagonal scatter, no zero fill) against
the slot-addressed COO route (fdb_plan_create_coo with FDB_J_SLOTS on the findstructralnz lists) on the same buffer.

    python scripts/diagonals_bench.py [--out FILE] [--n 10000000] [--rounds 3]

f is the native tridiagonal fdbs_tridiag, coloured cyclically by matrix_colors.  Workloads, forward and central:
  bidiagonal   a Bidiagonal :U target (2n-1 slots, 2 colours) through the mirror;
  tridiagonal  a Tridiagonal-layout buffer [dl; d; du] (3n-2 slots, 3 colours) through FDB_J_DIAGONALS at the C ABI,
               against the mirror's Tridiagonal route (the COO slot route).
Per workload and mode, the two arms run in alternating rounds and each number is the best round:
  plan_s       host wall time of the plan build; the COO arm's includes its host entry lists (findstructralnz);
  step_ms      one whole Jacobian, CUDA events on the stream over more than a second of calls; spread over the rounds;
  scatter_ms   the scatter per call from fdb_plan_enable_timing (the COO arm's zero fill of J is not inside it);
  bytes        the scatter's compulsory traffic: 8*j_len written + 8*n*(C+1) read forward / 8*n*2C central (every f!
               output row once; the COO arm adds 13 bytes of index and colour streams per entry);
  share_store / share_stream   the scatter's GB/s by that model over fdbs_store_probe / fdbs_stream_probe 1:1 measured
               in the same run.
Both arms' J are compared bit for bit.  Prints one JSON line; the card's name, power limit and max SM clock are read in
the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path


ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import _bootstrap  # noqa: E402

FD = {"forward": 0, "central": 1}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


def timed(fn, min_s=1.0):
    """per-call device time over at least min_s of calls"""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(3, int(min_s / max(time.perf_counter() - t0, 1e-6)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def scatter_ms(plan, fn, reps=20):
    plan.enable_timing(True)
    plan.read_timing()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    ms, launches = plan.read_timing()
    plan.enable_timing(False)
    return ms / reps, launches / reps


def probes(pkg, nbytes):
    S = pkg._lib.synth()
    n = int(nbytes // 8)
    src = torch.empty(n + 8, dtype=torch.float64, device="cuda").uniform_()
    dst = torch.empty(n + 8, dtype=torch.float64, device="cuda")
    sink = torch.zeros(1, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"store": 0.0, "stream_1:1": 0.0}
    h = (n // 2) & ~1                        # the stream probe wants even leading dimensions
    for blocks in (sms * 4, sms * 8, sms * 16):
        assert S.fdbs_store_probe(dst.data_ptr(), n, 0, blocks, None) == 0
        assert S.fdbs_stream_probe(src.data_ptr(), h, 1, dst.data_ptr(), h, 1, h, blocks, sink.data_ptr(), None) == 0
        ms = timed(lambda: S.fdbs_store_probe(dst.data_ptr(), n, 0, blocks, None), 0.3)
        out["store"] = max(out["store"], 8.0 * n / (ms * 1e-3) / 1e9)
        ms = timed(lambda: S.fdbs_stream_probe(src.data_ptr(), h, 1, dst.data_ptr(), h, 1, h, blocks, sink.data_ptr(),
                                               None), 0.3)
        out["stream_1:1"] = max(out["stream_1:1"], 16.0 * h / (ms * 1e-3) / 1e9)
    return out


def coo_plan(pkg, api, sp, jlen, cv, fdtype):
    """the slot-addressed route: host entry lists, then fdb_plan_create_coo (timed together)"""
    L = pkg._lib
    t0 = time.perf_counter()
    rows, cols, slots = sp.findstructralnz()
    o = api._opts(FD[fdtype], 0)
    cv_ptr, keep = api._index_ptr(cv)
    h = C.c_void_p()
    L.check(L.lib().fdb_plan_create_coo(C.byref(h), sp.n, sp.n, len(rows), rows.ctypes.data, cols.ctypes.data,
                                        L.FDB_J_SLOTS, slots.ctypes.data, jlen, cv_ptr, C.byref(o)))
    torch.cuda.synchronize()
    return pkg.Plan(h.value, (keep, rows, cols, slots)), time.perf_counter() - t0


def diag_plan(pkg, api, n, l, u, jlen, cv, fdtype):
    """FDB_J_DIAGONALS at the C ABI"""
    L = pkg._lib
    t0 = time.perf_counter()
    o = api._opts(FD[fdtype], 0)
    cv_ptr, keep = api._index_ptr(cv)
    h = C.c_void_p()
    L.check(L.lib().fdb_plan_create_banded(C.byref(h), n, n, l, u, L.FDB_J_DIAGONALS, jlen, cv_ptr, C.byref(o)))
    torch.cuda.synchronize()
    return pkg.Plan(h.value, (keep,)), time.perf_counter() - t0


def runner(pkg, J, f, x, fdtype, cv, plan):
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    cache.plan_for = lambda *a: plan
    return lambda: pkg.finite_difference_jacobian_(J, f, x, cache)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import api
    L = pkg._lib
    dev = torch.device("cuda", 0)
    n = args.n
    x = torch.empty(n, dtype=torch.float64, device=dev)
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0xD1A6, None)
    ctx = L.TridiagCtx(n, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    res = {"card": card(), "n": n, "workloads": {}}
    pr = probes(pkg, 8 * (3 * n - 2))
    res["probe_GBps"] = pr
    for wl in ("bidiagonal", "tridiagonal"):
        for fdtype in ("forward", "central"):
            if wl == "bidiagonal":
                l, u = 0, 1
                Jn, Jc = pkg.Bidiagonal(n, "U", device=dev), pkg.Bidiagonal(n, "U", device=dev)
            else:
                l, u = 1, 1
                Jn, Jc = pkg.Tridiagonal(n, device=dev), pkg.Tridiagonal(n, device=dev)
            jlen = Jn.buf.numel()
            cv = pkg.matrix_colors(Jn)
            Cc = int(cv.max())
            r = {"j_len": jlen, "n_colors": Cc}
            best = {"new": {}, "coo": {}}
            for _ in range(args.rounds):
                for arm in ("new", "coo"):
                    if arm == "new":
                        if wl == "bidiagonal":
                            t0 = time.perf_counter()
                            plan = api.make_plan(Jn, Jn, cv, fdtype, n, dev)
                            torch.cuda.synchronize()
                            ps = time.perf_counter() - t0
                        else:
                            plan, ps = diag_plan(pkg, api, n, l, u, jlen, cv, fdtype)
                        J = Jn
                    else:
                        plan, ps = coo_plan(pkg, api, Jc, jlen, cv, fdtype)
                        J = Jc
                    step = runner(pkg, J, f, x, fdtype, cv, plan)
                    st = timed(step)
                    sc, launches = scatter_ms(plan, step)
                    b = best[arm]
                    b.setdefault("plan_s", []).append(ps)
                    b.setdefault("step_ms", []).append(st)
                    b.setdefault("scatter_ms", []).append(sc)
                    b["scatter_launches"] = launches
                    b["jkind"] = plan.info()["jkind"]
                    plan.destroy()
            reads = 8 * n * (Cc + 1) if fdtype == "forward" else 8 * n * 2 * Cc
            for arm, b in best.items():
                out = {k: min(v) for k, v in b.items() if isinstance(v, list)}
                out["step_spread"] = (max(b["step_ms"]) - min(b["step_ms"])) / min(b["step_ms"])
                out["jkind"], out["scatter_launches"] = b["jkind"], b["scatter_launches"]
                out["bytes"] = 8 * jlen + reads + (13 * jlen if arm == "coo" else 0)
                gbps = out["bytes"] / (out["scatter_ms"] * 1e-3) / 1e9
                out["scatter_GBps"] = gbps
                out["share_store"] = gbps / pr["store"]
                out["share_stream"] = gbps / pr["stream_1:1"]
                r[arm] = out
            r["step_speedup"] = r["coo"]["step_ms"] / r["new"]["step_ms"]
            r["bit_identical"] = bool(torch.equal(Jn.buf.view(torch.int64), Jc.buf.view(torch.int64)))
            res["workloads"][f"{wl}_{fdtype}"] = r
            del Jn, Jc
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
