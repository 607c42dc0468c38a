"""Out-of-place CSR Jacobians: the CSR result (fdb_oop_plan_create_csr) against what a caller who needs CSR had before it,
on the same problem:
  csr       the CSR plan with every f! output resident: the fused CSR compaction (oop_compact_csr) forms the quotients;
  csr_copy  the same plan kind with one f! output per group (max_batch 1, a small scratch budget): the CSR scatter writes
            the candidates and the kCopy compaction (oop_compact<false, kCopy> over colval and rowptr) drops the zeros;
  csc_conv  the CSC route's sparse result (fdb_oop_plan_create_csc, FDB_OOP_SPARSE), its kept count read back, then a
            device CSC -> CSR conversion of the result: torch's sparse_csc_tensor(...).to_sparse_csr() (named in the output
            as `conversion`; it sorts on the device; a stable device sort by row is the fallback when torch does not
            convert CSC on the device).  Its kernels are conv_ms; the kept count is read back on the host before it.

    python scripts/oop_csr_bench.py [--out FILE] [--workloads c2,c4,stencil] [--modes forward,central]

Workloads (the patterns, colourings, x and native f of scripts/csr_bench.py, rows with sorted columns): c2 (N = 10^7
tridiagonal, 3 colours, fdbs_tridiag), c4 (N = 5*10^6, 8 random columns per row, 64 colours, fdbs_ellrows), stencil
(g = 1000 5-point stencil, 5 colours, fdbs_lap5).
Per arm: plan_s (host wall time of the plan build, the host work the arm needs included); step_ms (one whole call,
CUDA events over more than a second of calls, best of three rounds, with its spread); from a torch.profiler trace of a run
of its own, compact_ms (the compaction kernel), conv_ms (csc_conv: the conversion's kernels) and library_ms (every
library kernel of the call: the fdb:: kernels and memsets).  compact_bytes is the fused CSR compaction's byte model
(compaction_bytes below) and compact_GBps that over compact_ms, against fdbs_stream_probe's best (1 read, 1 write) rate
measured in the same run (probe_share); compact_bytes counts the reads per candidate, and
compact_bytes_compulsory / probe_share_compulsory count forward-mode f(x) once per row, the compulsory traffic.  Every
arm's step reads the kept count back to the host, as finite_difference_jacobian does.  Results are bit-compared across
arms (rowptr, colval, values).  Prints one JSON line with the card's name, power limit and max SM clock, read in the
same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np
import scipy.sparse as sp

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

import torch  # noqa: E402

import _bootstrap  # noqa: E402
from csr_bench import card, stream_probe_gbps, timed, workload  # noqa: E402


def compaction_bytes(m, n, E, kept, mode, color_bytes, cyclic, compulsory=False):
    """Bytes of the fused CSR compaction.  Reads: colval (4 B per candidate), the staged row pointer (4 B per row), the
    colour table (unless the colouring is cyclic), and per candidate its slab element and its f(x) element (central: the
    plus and the minus slab element).  Writes: 16 B per kept entry (column and value) and 8 B per row-pointer entry.
    compulsory: forward-mode f(x) counted once per row instead of once per candidate (every candidate of a row reads the
    same f(x) element, so the gathers are row-local); with a valid colouring every slab element is read once."""
    fx = 8 * m if compulsory and mode == "forward" else 8 * E
    reads = 4 * E + 4 * (m + 1) + (0 if cyclic else color_bytes * n) + 8 * E + fx
    writes = 16 * kept + 8 * (m + 1)
    return reads + writes


def traced(fn, reps=10):
    """{kernel name: device ms per call} from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_time > 0:
            out[e.name] = out.get(e.name, 0.0) + e.device_time / reps / 1e3
    return out


def is_f(name):
    """a kernel of the synthetic f (synth_fns.cu keeps them in an anonymous namespace)"""
    return "(anonymous namespace)::k_" in name


def sum_of(tr, pred):
    v = [t for k, t in tr.items() if pred(k)]
    return float(sum(v)) if v else None


def convert_csc_to_csr(m, n, colptr, rowval, nzval, nnz, how):
    """device CSC -> CSR of a kept-entry result (0-based int64 indices)"""
    if how == "torch.to_sparse_csr":
        T = torch.sparse_csc_tensor(colptr - 1, rowval[:nnz] - 1, nzval[:nnz], size=(m, n))
        R = T.to_sparse_csr()
        return R.crow_indices() + 1, R.col_indices() + 1, R.values()
    cols = torch.repeat_interleave(torch.arange(n, device=colptr.device), torch.diff(colptr))
    rows = rowval[:nnz] - 1
    o = torch.sort(rows, stable=True).indices
    rp = torch.ones(m + 1, dtype=torch.int64, device=colptr.device)
    rp[1:] += torch.cumsum(torch.bincount(rows, minlength=m), 0)
    return rp, cols[o] + 1, nzval[:nnz][o]


def run_mode(pkg, api, A, cv, x, faddr, fctx, mode, probe):
    L = pkg._lib
    lib = L.lib()
    m, n = A.shape
    E = A.nnz
    code = L.FDB_CENTRAL if mode == "central" else L.FDB_FORWARD
    res = {}
    ref = None
    for arm in ("csr", "csr_copy", "csc_conv"):
        kw = {"max_batch": 1, "scratch_bytes": 8 * (m + 2) * (2 if mode == "central" else 1) + 64} if arm == "csr_copy" \
            else {"max_batch": 64}
        opts = api._opts(code, 0, **kw)
        t0 = time.perf_counter()
        if arm == "csc_conv":
            T = A.tocsc()
            cp, rv = T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1
            h = api._new_handle("fdb_oop_plan_create_csc", m, n, cp.ctypes.data, rv.ctypes.data, cv.ctypes.data,
                                L.FDB_OOP_SPARSE, m, C.byref(opts))
            del T, cp, rv
        else:
            rp, cl = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
            h = api._new_handle("fdb_oop_plan_create_csr", m, n, rp.ctypes.data, cl.ctypes.data, cv.ctypes.data,
                                L.FDB_OOP_SPARSE, m, C.byref(opts))
            del rp, cl
        plan = api.Plan(h.value)
        torch.cuda.synchronize()
        r = {"plan_s": time.perf_counter() - t0}
        info = plan.info()
        r["n_groups"] = info["n_groups"]
        ptr = torch.empty((m if arm != "csc_conv" else n) + 1, dtype=torch.int64, device="cuda")
        idx = torch.empty(E, dtype=torch.int64, device="cuda")
        val = torch.empty(E, dtype=torch.float64, device="cuda")
        nnz = torch.empty(1, dtype=torch.int64, device="cuda")
        out = L.OopOut()
        out.colptr, out.rowval, out.nzval, out.cap, out.nnz = ptr.data_ptr(), idx.data_ptr(), val.data_ptr(), E, \
            nnz.data_ptr()
        how = None
        if arm == "csc_conv":
            how = "torch.to_sparse_csr"
            try:
                L.check(lib.fdb_jacobian_oop(plan._h, faddr, C.addressof(fctx), x.data_ptr(), C.byref(out), None, None,
                                             L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, None))
                k = int(nnz.item())
                convert_csc_to_csr(m, n, ptr, idx, val, k, how)
            except (RuntimeError, NotImplementedError):
                how = "torch.sort by row (stable)"
            r["conversion"] = how
        conv = [None]

        def step():
            # every arm reads the kept count back, as finite_difference_jacobian does to size its result
            L.check(lib.fdb_jacobian_oop(plan._h, faddr, C.addressof(fctx), x.data_ptr(), C.byref(out), None, None,
                                         L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, None))
            k = int(nnz.item())
            if how is not None:
                conv[0] = convert_csc_to_csr(m, n, ptr, idx, val, k, how)
        r["step_ms"], r["step_spread"] = timed(step)
        tr = traced(step)
        r["compact_ms"] = sum_of(tr, lambda k: "oop_compact" in k)
        r["library_ms"] = sum_of(tr, lambda k: "fdb::" in k or "Memset" in k)
        r["kernels"] = {k: round(v, 5) for k, v in sorted(tr.items(), key=lambda kv: -kv[1])[:12]}
        kept = int(nnz.item())
        if how is not None:
            r["conv_ms"] = sum_of(tr, lambda k: not ("fdb::" in k or "Memset" in k or is_f(k)))
            got = tuple(t.clone() for t in conv[0])
        else:
            got = (ptr.clone(), idx[:kept].clone(), val[:kept].clone())
        r["kept"] = kept
        if arm == "csr":
            r["compact_bytes"] = compaction_bytes(m, n, E, kept, mode, info["color_bits"] // 8, cv_cyclic(cv))
            if r["compact_ms"]:
                r["compact_GBps"] = r["compact_bytes"] / (r["compact_ms"] * 1e-3) / 1e9
                r["probe_share"] = r["compact_GBps"] / probe
                r["compact_bytes_compulsory"] = compaction_bytes(m, n, E, kept, mode, info["color_bits"] // 8,
                                                                 cv_cyclic(cv), compulsory=True)
                r["probe_share_compulsory"] = r["compact_bytes_compulsory"] / (r["compact_ms"] * 1e-3) / 1e9 / probe
            ref = got
        else:
            r["bit_identical_to_csr"] = bool(torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]) and
                                             torch.equal(got[2].view(torch.int64), ref[2].view(torch.int64)))
        res[arm] = r
        del plan, ptr, idx, val, nnz, conv, got
        torch.cuda.empty_cache()
    return res


def cv_cyclic(cv):
    C_ = int(cv.max())
    return bool(C_ > 0 and np.array_equal(cv, np.arange(len(cv)) % C_ + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--workloads", default="c2,c4,stencil")
    ap.add_argument("--modes", default="forward,central")
    args = ap.parse_args()
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import api
    probe = stream_probe_gbps(pkg, 1 << 27)
    res = {"card": card(), "stream_probe_GBps": probe, "workloads": {}}
    for w in args.workloads.split(","):
        A, cv, x, faddr, fctx, keep = workload(pkg, w)
        res["workloads"][w] = {"n": A.shape[1], "nnz": A.nnz, "n_colors": int(cv.max()),
                               "modes": {md: run_mode(pkg, api, A, cv, x, faddr, fctx, md, probe)
                                         for md in args.modes.split(",")}}
        del A, x, keep
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
