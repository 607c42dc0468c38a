"""CSR Jacobians: the CSR plan (fdb_plan_create_csr, J = the CSR's nzval) against the two routes a caller had before it,
on the same problem:
  coo      the COO slot route (fdb_plan_create_coo, FDB_J_SLOTS, slots 1..nnz) on the same buffer, with its zero fill;
  csc      the CSC route (fdb_plan_create_csc on the CSC of the same matrix), J left in CSC order;
  csc_perm the CSC route plus a gather of its nzval into CSR order through a precomputed permutation (one index_select
           into a second J-sized buffer): the cheapest conversion a caller could write.

    python scripts/csr_bench.py [--out FILE] [--workloads c2,c4,stencil]

Workloads (forward mode, the library's default step sizes):
  c2       N = 10^7 tridiagonal, 3 cyclic colours, f = fdbs_tridiag;
  c4       N = 5*10^6, 8 random columns per row, 64 colours (bench.py's C4 instance), f = fdbs_ellrows;
  stencil  g = 1000 2-D 5-point stencil (N = 10^6), 5 colours, f = fdbs_lap5.
Per arm: plan_s (host wall time of the plan build, including the host work the arm needs: the COO entry list, the CSC
and the permutation); step_ms (one whole Jacobian, CUDA events over more than a second of calls, best of three rounds;
spread = (max - min) / min); scatter_ms and fill_ms per call from a torch.profiler trace of their own run (the csc_perm
arm's gather is in gather_ms).  For the CSR plan, moved_GBps = fdb_plan_info's moved_bytes_scatter over its scatter time
and probe_share = that over fdbs_stream_probe's best (1 read, 1 write) rate measured in the same run.  Every arm's J is
bit-compared with the CSR plan's (in CSR order).  Prints one JSON line with the card's name, power limit and max SM
clock, read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import scipy.sparse as sp

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
    """device time per call of the kernels whose name contains one of `names`, from torch.profiler"""
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


def stream_probe_gbps(pkg, n):
    """best (1 read, 1 write) streaming rate in GB/s (bytes read + written)"""
    S = pkg._lib.synth()
    src = torch.ones(n, dtype=torch.float64, device="cuda")
    dst = torch.empty(n, dtype=torch.float64, device="cuda")
    sink = torch.zeros(1, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    best = 0.0
    for blocks in (sms * 4, sms * 8, sms * 16):
        ms, _ = timed(lambda: S.fdbs_stream_probe(src.data_ptr(), n, 1, dst.data_ptr(), n, 1, n, blocks, sink.data_ptr(),
                                                  None), 0.3, 2)
        best = max(best, 16.0 * n / (ms * 1e-3) / 1e9)
    return best


def workload(pkg, name):
    """(scipy CSR pattern with sorted columns, colorvec, x, f address, f ctx, keepalive)"""
    L = pkg._lib
    S = L.synth()
    if name == "c2":
        n = 10_000_000
        A = sp.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csr", dtype=np.int8)
        cv = (np.arange(n) % 3 + 1).astype(np.int64)
        ctx, fn, keep = L.TridiagCtx(n, 0), S.fdbs_tridiag, ()
    elif name == "c4":
        import bench
        n, K, Cc = bench.C4_N, bench.C4_K, bench.C4_C
        d_cols, d_coef = bench.c4_instance_torch(torch.device("cuda"), n, K, Cc)
        cols = d_cols.cpu().numpy()
        rows = np.tile(np.arange(n, dtype=np.int32), K)
        A = sp.csr_matrix((np.ones(n * K, np.int8), (rows, cols.reshape(-1))), shape=(n, n))
        cv = (np.arange(n) % Cc + 1).astype(np.int64)
        ctx, fn, keep = L.EllCtx(n, K, d_cols.data_ptr(), d_coef.data_ptr(), 0), S.fdbs_ellrows, (d_cols, d_coef)
    else:
        g = 1000
        n = g * g
        T = sp.diags([np.ones(g - 1), np.ones(g), np.ones(g - 1)], [-1, 0, 1], format="csr", dtype=np.int8)
        A = (sp.kron(sp.identity(g, dtype=np.int8), T) + sp.kron(T, sp.identity(g, dtype=np.int8))).tocsr()
        idx = np.arange(n)
        cv = (((idx % g) + 2 * (idx // g)) % 5 + 1).astype(np.int64)
        ctx, fn, keep = L.Lap5Ctx(g, 0), S.fdbs_lap5, ()
    A.sort_indices()
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    S.fdbs_fill_x(x.data_ptr(), n, 0xC5A, None)
    return A, cv, x, C.cast(fn, C.c_void_p).value, ctx, keep


def run_workload(pkg, api, name, probe):
    L = pkg._lib
    lib = L.lib()
    A, cv, x, faddr, fctx, keep = workload(pkg, name)
    m, n = A.shape
    nnz = A.nnz
    opts = api._opts(L.FDB_FORWARD, 0)
    res = {"n": n, "nnz": nnz, "n_colors": int(cv.max()), "arms": {}}
    ref = None
    for arm in ("csr", "coo", "csc", "csc_perm"):
        t0 = time.perf_counter()
        gather = None
        if arm == "csr":
            rp, cl = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
            h = api._new_handle("fdb_plan_create_csr", m, n, rp.ctypes.data, cl.ctypes.data, cv.ctypes.data, C.byref(opts))
            kern = "diff_scatter_csr"
            del rp, cl
        elif arm == "coo":
            coo = A.tocoo()
            rows, cols = coo.row.astype(np.int64) + 1, coo.col.astype(np.int64) + 1
            slots = np.arange(1, nnz + 1, dtype=np.int64)
            h = api._new_handle("fdb_plan_create_coo", m, n, nnz, rows.ctypes.data, cols.ctypes.data, L.FDB_J_SLOTS,
                                slots.ctypes.data, nnz, cv.ctypes.data, C.byref(opts))
            kern = "diff_scatter_dest"
            del coo, rows, cols, slots
        else:
            T = sp.csr_matrix((np.arange(nnz, dtype=np.float64), A.indices, A.indptr), shape=A.shape).tocsc()
            cp, rv = T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1
            h = api._new_handle("fdb_plan_create_csc", m, n, cp.ctypes.data, rv.ctypes.data, L.FDB_J_CSC_NZVAL, None, None,
                                0, cv.ctypes.data, C.byref(opts))
            kern = "diff_scatter"
            if arm == "csc_perm":
                # CSR slot s holds CSC slot inv[s]
                inv = np.empty(nnz, np.int64)
                inv[T.data.astype(np.int64)] = np.arange(nnz, dtype=np.int64)
                gather = torch.from_numpy(inv).cuda()
                del inv
            del T, cp, rv
        plan = api.Plan(h.value)
        torch.cuda.synchronize()
        r = {"plan_s": time.perf_counter() - t0}
        info = plan.info()
        r.update(fcalls=info["fcalls_per_jacobian"], moved_bytes_scatter=info["moved_bytes_scatter"])
        J = torch.full((nnz,), float("nan"), dtype=torch.float64, device="cuda")
        Jcsr = torch.empty(nnz, dtype=torch.float64, device="cuda") if gather is not None else None

        def step():
            L.check(lib.fdb_jacobian(plan._h, faddr, C.addressof(fctx), x.data_ptr(), J.data_ptr(), None, None,
                                     L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, None))
            if gather is not None:
                torch.index_select(J, 0, gather, out=Jcsr)
        r["step_ms"], r["step_spread"] = timed(step)
        tr = traced_ms(step, [kern, "Memset", "ndex"])
        r["scatter_ms"], r["fill_ms"] = tr[kern], tr["Memset"]
        if gather is not None:
            r["gather_ms"] = tr["ndex"]
        if arm == "csr" and r["scatter_ms"]:
            r["moved_GBps"] = info["moved_bytes_scatter"] / (r["scatter_ms"] * 1e-3) / 1e9
            r["probe_share"] = r["moved_GBps"] / probe
        got = (Jcsr if gather is not None else J)
        if arm == "csr":
            ref = got.clone()
        elif arm != "csc":          # the csc arm's J is in CSC order: its values are checked by the csc_perm arm
            r["bit_identical_to_csr"] = bool(torch.equal(got.view(torch.int64), ref.view(torch.int64)))
        res["arms"][arm] = r
        del J, Jcsr, plan, gather
        torch.cuda.empty_cache()
    del keep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--workloads", default="c2,c4,stencil")
    args = ap.parse_args()
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import api
    probe = stream_probe_gbps(pkg, 1 << 27)
    res = {"card": card(), "stream_probe_GBps": probe, "workloads": {}}
    for w in args.workloads.split(","):
        res["workloads"][w] = run_workload(pkg, api, w, probe)
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
