"""BlockBandedMatrix Jacobians in BlockBandedMatrices' storage: the block-dense plan (fdb_plan_create_block_dense)
against the slot-addressed route (fdb_plan_create_coo with FDB_J_SLOTS on the same buffer) and the padded route (the
mirror's BlockBandedMatrix, a BandedBlockBandedMatrix with sub-block bandwidths (b-1, b-1), through
fdb_plan_create_block_banded), on the same problem.

    python scripts/block_dense_bench.py [--out FILE] [--nblocks 250000] [--b 8]

Problem: nblocks square blocks of b, block bandwidths l = u = 1 (n = nblocks*b; 4.8e7 slots at the defaults), f =
fdbs_ellrows with every row reading every column of its block row's band (a Jacobian that fills the structure).  Each
route uses its own matrix_colors: (l+u+1)*b colours for the compact storage (the slot route shares it), (l+u)(2b-1)+b
for the padded one.  Per route and mode (forward, central):
  plan_s       host wall time of the plan build (the slot route's includes findstructralnz on the host);
  step_ms      one whole Jacobian through the C ABI (f(x), step sizes, the colours' f! calls, the scatter), CUDA events
               over more than a second of calls, best of three rounds; spread = (max - min) / min of the rounds;
  scatter_ms   the scatter kernel per call, and fill_ms the zero fill of J per call (the slot route), from a
               torch.profiler trace of their own run;
  fcalls       f! points per Jacobian; slots_written = J doubles the scatter stores per call;
  store_share  the scatter's stores (8 bytes per slot written) per second over fdbs_store_probe measured in the same run.
The compact result is bit-compared with the slot route's.  Prints one JSON line with the card's name, power limit and
max SM clock, read in the same run."""
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


def traced_ms(fn, names, reps=10):
    """median device time per call of the kernels whose name contains one of `names`, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for nm in names:
        ts = [e.device_time for e in prof.events() if nm in e.name and e.device_time > 0]
        out[nm] = float(np.sum(ts)) / reps / 1e3 if ts else None
    return out


def store_probe_gbps(pkg, n):
    S = pkg._lib.synth()
    dst = torch.empty(n + 8, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    best = 0.0
    for blocks in (sms * 4, sms * 8, sms * 16):
        ms, _ = timed(lambda: S.fdbs_store_probe(dst.data_ptr(), n, 0, blocks, None), 0.3, 2)
        best = max(best, 8.0 * n / (ms * 1e-3) / 1e9)
    return best


class EllF:
    """fdbs_ellrows: row i of block row K reads every column of block columns K-l .. K+u (uniform blocks of b)"""

    def __init__(self, pkg, N, b, l, u, seed=7):
        L = pkg._lib
        n = N * b
        K = (l + u + 1) * b
        krow = np.arange(n) // b
        c0 = np.maximum(krow - l, 0) * b
        width = (np.minimum(krow + u, N - 1) + 1) * b - c0
        p = np.arange(K)[:, None]
        cols = np.where(p < width[None, :], c0[None, :] + p, c0[None, :]).astype(np.int32)
        coef = np.random.default_rng(seed).uniform(-1, 1, size=(K, n)) * (p < width[None, :])
        self.d_cols = torch.from_numpy(np.ascontiguousarray(cols)).cuda()
        self.d_coef = torch.from_numpy(np.ascontiguousarray(coef)).cuda()
        self.ctx = L.EllCtx(n, K, self.d_cols.data_ptr(), self.d_coef.data_ptr(), 0)
        self.addr = C.cast(L.synth().fdbs_ellrows, C.c_void_p).value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--nblocks", type=int, default=250_000)
    ap.add_argument("--b", type=int, default=8)
    args = ap.parse_args()
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import api
    L = pkg._lib
    lib = L.lib()
    N, b, l, u = args.nblocks, args.b, 1, 1
    n = N * b
    rb = [b] * N
    blocks = np.asarray(rb, np.int64)
    res = {"card": card(), "nblocks": N, "b": b, "l": l, "u": u, "n": n, "routes": {}}
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0xB10C, None)
    f = EllF(pkg, N, b, l, u)
    fctx = C.addressof(f.ctx)
    S = pkg.BlockSkylineMatrix(rb, rb, (l, u), device="cpu", data=torch.empty(0))
    P = pkg.BlockBandedMatrix(rb, rb, (l, u), device="cpu", data=torch.empty(0))
    res["j_len_compact"], res["j_len_padded"] = S.j_len, P.w * P.n
    cv_s, cv_p = S.matrix_colors(), P.matrix_colors()
    probe = store_probe_gbps(pkg, S.j_len)
    res["store_probe_GBps"] = probe
    for fd_name, fd in (("forward", L.FDB_FORWARD), ("central", L.FDB_CENTRAL)):
        opts = api._opts(fd, 0)
        out = {}
        results = {}
        for route in ("compact", "slots", "padded"):
            t0 = time.perf_counter()
            if route == "compact":
                h = api._new_handle("fdb_plan_create_block_dense", N, blocks.ctypes.data, l, u, S.j_len, cv_s.ctypes.data,
                                    C.byref(opts))
                jlen, kern = S.j_len, "diff_scatter_block_dense"
            elif route == "slots":
                rows, cols, slots = S.findstructralnz()
                h = api._new_handle("fdb_plan_create_coo", n, n, len(rows), rows.ctypes.data, cols.ctypes.data,
                                    L.FDB_J_SLOTS, slots.ctypes.data, S.j_len, cv_s.ctypes.data, C.byref(opts))
                del rows, cols, slots
                jlen, kern = S.j_len, "diff_scatter_dest"
            else:
                h = api._new_handle("fdb_plan_create_block_banded", N, blocks.ctypes.data, l, u, P.lam, P.mu, P.w * P.n,
                                    cv_p.ctypes.data, C.byref(opts))
                jlen, kern = P.w * P.n, "diff_scatter_block_band"
            plan = api.Plan(h.value)
            torch.cuda.synchronize()
            r = {"plan_s": time.perf_counter() - t0}
            info = plan.info()
            r.update(n_colors=info["n_colors"], fcalls=info["fcalls_per_jacobian"], slots_written=info["j_len"],
                     n_entries=info["n_entries"])
            J = torch.full((jlen,), float("nan"), dtype=torch.float64, device="cuda")

            def step():
                L.check(lib.fdb_jacobian(plan._h, f.addr, fctx, x.data_ptr(), J.data_ptr(), None, None,
                                         L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, None))
            r["step_ms"], r["step_spread"] = timed(step)
            tr = traced_ms(step, [kern, "Memset"])
            r["scatter_kernel"], r["scatter_ms"], r["fill_ms"] = kern, tr[kern], tr["Memset"]
            if r["scatter_ms"]:
                r["store_GBps"] = 8.0 * jlen / (r["scatter_ms"] * 1e-3) / 1e9
                r["store_share"] = r["store_GBps"] / probe
            c0 = f.ctx.calls
            step()
            torch.cuda.synchronize()
            r["fcalls_counted"] = f.ctx.calls - c0
            if route != "padded":
                results[route] = J.clone()
            out[route] = r
            del J, plan
            torch.cuda.empty_cache()
        out["compact_bit_identical_to_slots"] = bool(torch.equal(results["compact"].view(torch.int64),
                                                                 results["slots"].view(torch.int64)))
        res["routes"][fd_name] = out
        del results
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
