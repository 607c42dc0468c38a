"""Block-banded Jacobians at PDE scale: the closed-form plan (fdb_plan_create_block_banded) against the slot-addressed
route it replaces (fdb_plan_create_coo on the entry list of findstructralnz), on the 5-point stencil of fdbs_lap5.

    python scripts/block_banded_bench.py [--out FILE] [--grids 1000,3000] [--coo-grid 1000]

J is a BandedBlockBandedMatrix with g blocks of g, l = u = lam = mu = 1 (9 slots per column), coloured by
matrix_colors (9 colours), forward mode.  Per grid:
  plan_s         host wall time of the mirror's plan build (the COO route's includes findstructralnz), coo-grid only for
                 the COO route: its host work grows with the entry count;
  step_ms        one whole Jacobian (f(x), the step sizes, the 9 colours and the scatter), CUDA events on the stream over
                 more than a second of calls, best of three rounds; spread = (max - min) / min of the rounds;
  scatter_ms     the scatter kernel per call, from a torch.profiler trace of its own run;
  bytes          the scatter's compulsory traffic from the model below; GB/s = bytes / scatter_ms;
  share_store / share_stream   the scatter's GB/s over fdbs_store_probe (pure stores) and fdbs_stream_probe 1:1
                 measured in the same run;
  group          GroupJacobian over [0, 0] against the single plan (step_ms of both), each result bit-compared with the
                 COO route's (coo-grid) or with the single plan's.
Byte model of the scatter: 8*w*n written (every slot once) + 8*n*(C + 1) read (each colour's f! output and f(x) once;
the gathers re-read rows from L2).  Prints one JSON line; the card's name, power limit and max SM clock are read in the
same run.  With one visible GPU the [0, 0] group shows the group's overhead only: scaling over distinct GPUs is not
measured."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import _bootstrap  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


def timed(fn, min_s=1.0, rounds=3):
    """best and spread of per-call device time over `rounds` rounds of at least min_s each"""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(3, int(min_s / max(time.perf_counter() - t0, 1e-6)))
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return min(out), (max(out) - min(out)) / min(out)


def kernel_ms(fn, name, reps=10):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if name in e.name and e.device_time > 0]
    return float(np.median(ts)) / 1e3 if ts else None, len(ts)


def probes(pkg, nbytes):
    S = pkg._lib.synth()
    n = int(nbytes // 8)
    src = torch.empty(n + 8, dtype=torch.float64, device="cuda").uniform_()
    dst = torch.empty(n + 8, dtype=torch.float64, device="cuda")
    sink = torch.zeros(1, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"store": 0.0, "stream_1:1": 0.0}
    for blocks in (sms * 4, sms * 8, sms * 16):
        ms, _ = timed(lambda: S.fdbs_store_probe(dst.data_ptr(), n, 0, blocks, None), 0.3, 2)
        out["store"] = max(out["store"], 8.0 * n / (ms * 1e-3) / 1e9)
        ms, _ = timed(lambda: S.fdbs_stream_probe(src.data_ptr(), n // 2, 1, dst.data_ptr(), n // 2, 1, n // 2, blocks,
                                                  sink.data_ptr(), None), 0.3, 2)
        out["stream_1:1"] = max(out["stream_1:1"], 8.0 * n / (ms * 1e-3) / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--grids", default="1000,3000")
    ap.add_argument("--coo-grid", type=int, default=1000, dest="coo_grid")
    args = ap.parse_args()
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import api, distributed
    L = pkg._lib
    dev = torch.device("cuda", 0)
    res = {"card": card(), "gpus_visible": torch.cuda.device_count(), "grids": {}}
    for g in [int(v) for v in args.grids.split(",")]:
        n = g * g
        r = {"n": n}
        B = pkg.BandedBlockBandedMatrix([g] * g, [g] * g, (1, 1), (1, 1), device=dev)
        cv = B.matrix_colors()
        x = torch.empty(n, dtype=torch.float64, device=dev)
        L.synth().fdbs_fill_x(x.data_ptr(), n, 0x1AB5, None)
        ctx = L.Lap5Ctx(g, 0)
        f = pkg.NativeFn(C.cast(L.synth().fdbs_lap5, C.c_void_p).value, ctx)
        t0 = time.perf_counter()
        cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B)
        plan = cache.plan_for(B, B, cache.colorvec, n)
        torch.cuda.synchronize()
        r["plan_s"] = time.perf_counter() - t0
        info = plan.info()
        r["n_entries"], r["n_colors"] = info["n_entries"], info["n_colors"]
        step = lambda: pkg.finite_difference_jacobian_(B, f, x, cache)
        r["step_ms"], r["step_spread"] = timed(step)
        r["scatter_ms"], r["scatter_launches_traced"] = kernel_ms(step, "diff_scatter_block_band")
        w, Cc = 9, info["n_colors"]
        r["bytes"] = 8 * w * n + 8 * n * (Cc + 1)
        pr = probes(pkg, 8 * w * n)
        r["probe_GBps"] = pr
        if r["scatter_ms"]:
            gbps = r["bytes"] / (r["scatter_ms"] * 1e-3) / 1e9
            r["scatter_GBps"] = gbps
            r["share_store"] = gbps / pr["store"]
            r["share_stream"] = gbps / pr["stream_1:1"]
        J_new = B.data.clone()
        ref = None
        if g == args.coo_grid:
            Bc = pkg.BandedBlockBandedMatrix([g] * g, [g] * g, (1, 1), (1, 1), device=dev)
            saved = api._block_banded_plan_args
            api._block_banded_plan_args = lambda J, sp: None
            try:
                t0 = time.perf_counter()
                cc = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=Bc)
                cc.plan_for(Bc, Bc, cc.colorvec, n)
                torch.cuda.synchronize()
                r["coo_plan_s"] = time.perf_counter() - t0
            finally:
                api._block_banded_plan_args = saved
            stepc = lambda: pkg.finite_difference_jacobian_(Bc, f, x, cc)
            r["coo_step_ms"], r["coo_step_spread"] = timed(stepc)
            r["coo_scatter_ms"], _ = kernel_ms(stepc, "diff_scatter_dest")
            ref = Bc.data.clone()
            r["bit_identical_to_coo"] = bool(torch.equal(J_new.view(torch.int64), ref.view(torch.int64)))
            del cc, Bc
        # group [0, 0] against the single plan
        BG = pkg.BandedBlockBandedMatrix([g] * g, [g] * g, (1, 1), (1, 1), device=dev)
        ctxs = [L.Lap5Ctx(g, 0), L.Lap5Ctx(g, 0)]
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_lap5, C.c_void_p).value, c) for c in ctxs]
        gj = distributed.GroupJacobian(BG, cv, "forward", [0, 0])
        run_g = lambda: gj.run(fs, x)
        r["group00_step_ms"], r["group00_spread"] = timed(run_g)
        r["single_step_ms_same_round"], _ = timed(step, 1.0, 1)
        cmp = ref if ref is not None else J_new
        r["group00_bit_identical"] = bool(torch.equal(BG.data.view(torch.int64), cmp.view(torch.int64)))
        r["group00_compared_with"] = "coo_route" if ref is not None else "single_plan"
        gj.close()
        res["grids"][str(g)] = r
        del B, BG, cache, plan, J_new, ref
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
