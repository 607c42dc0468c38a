"""Dense Hessian on the device (fdb_hessian, src/hessians.jl:202-292): time, f-evaluations per second, batch-cap sweep,
the split between f and the library's kernels, and checks against the CPU restatement and the closed form.

    python scripts/hessian_bench.py [--out FILE]

f is the synthetic quartic of include/fdjac_synth.h (fdbs_quartic), whose Hessian is known in closed form.  Prints one
JSON line; the card's name and power limit are read in the same run."""
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
from scalar_oracle import fd_scalar_oracle as so  # noqa: E402

LIB_KERNELS = ("hess_patch", "hess_assemble", "component_eps", "replicate_x")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


class Problem:
    def __init__(self, pkg, n, seed=7):
        rng = np.random.default_rng(seed + n)
        self.n, self.a, self.w = n, 0.5 + rng.random(n), rng.random(n) * 2 - 1
        self.d_a, self.d_w = torch.from_numpy(self.a).cuda(), torch.from_numpy(self.w).cuda()
        self.x = torch.empty(n, dtype=torch.float64, device="cuda")
        pkg._lib.synth().fdbs_fill_x(self.x.data_ptr(), n, 0xC0FFEE + n, None)
        self.ctx = pkg._lib.ScalarCtx(n, self.d_a.data_ptr(), self.d_w.data_ptr(), 0)
        self.fn = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_quartic, C.c_void_p).value, self.ctx)
        self.H = pkg.zeros_colmajor(n, n)

    def closed_form_entries(self, x, rows, cols):
        v = self.w[rows] * self.w[cols] / self.n
        v = v + np.where(rows == cols, 12 * self.a[rows] * x[rows] ** 2, 0.0) + (np.abs(rows - cols) == 1)
        return v


def time_hessian(pkg, p, cache, reps):
    pkg.finite_difference_hessian_(p.H, p.fn, p.x, cache)          # warm-up (plan build, module load)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        pkg.finite_difference_hessian_(p.H, p.fn, p.x, cache)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def kernel_split(pkg, p, cache, out_dir):
    from torch.profiler import ProfilerActivity, profile
    pkg.finite_difference_hessian_(p.H, p.fn, p.x, cache)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pkg.finite_difference_hessian_(p.H, p.fn, p.x, cache)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        us[e.key] = us.get(e.key, 0.0) + e.device_time_total
    lib = {k: sum(v for name, v in us.items() if k in name) for k in LIB_KERNELS}
    f_us = sum(v for name, v in us.items() if "k_scalar" in name)
    return f_us / 1e6, {k: v / 1e6 for k, v in lib.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "hessian_bench needs a GPU"
    pkg = _bootstrap.load_package()
    so.build()
    res = {"metric": "hessian", "card": card(), "f": "fdbs_quartic"}

    # batch-cap sweep at n = 1000
    p = Problem(pkg, 1000)
    sweep = {}
    for mb in (64, 256, 1024, 4096, 16384):
        sweep[mb] = time_hessian(pkg, p, pkg.HessianCache(p.x, max_batch=mb), reps=2)
    res["max_batch_sweep_s_n1000"] = sweep
    best = min(sweep, key=sweep.get)
    res["best_max_batch"] = best

    for n in (1000, 2000):
        p = p if n == 1000 else Problem(pkg, n)
        cache = pkg.HessianCache(p.x, max_batch=best)
        t = time_hessian(pkg, p, cache, reps=3)
        pts = 2 * n * n + 1
        info = cache._last_plan.info()
        row = {"hessian_s": t, "f_evals_per_s": pts / t, "f_points": pts, "alg_bytes": info["alg_bytes_scatter"],
               "f_read_bytes": 8 * n * pts}
        f_s, lib = kernel_split(pkg, p, cache, None)
        row["f_kernel_s"], row["lib_kernel_s"] = f_s, lib
        patched = 2 * n + 8 * (n * (n - 1) // 2)
        asm_bytes = 8 * pts + 8 * n * n
        row["patch_bytes"], row["assemble_bytes"] = 16 * patched, asm_bytes
        if lib["hess_patch"] > 0:
            row["patch_GBps"] = 16 * patched / lib["hess_patch"] / 1e9
        if lib["hess_assemble"] > 0:
            row["assemble_GBps"] = asm_bytes / lib["hess_assemble"] / 1e9
        xh = p.x.cpu().numpy()
        Hd = p.H.cpu().numpy()
        if n == 1000:
            t0 = time.perf_counter()
            ref = so.hessian(so.SynthScalar(n, p.a, p.w).native("synth_quartic"), xh)
            row["cpu_oracle_s"] = time.perf_counter() - t0
            a, b = Hd.view(np.uint64), ref["H"].view(np.uint64)
            row["bit_identical_to_oracle"] = bool(np.array_equal(a, b))
            row["entries_differing"] = int(np.count_nonzero(a != b))
        else:
            rng = np.random.default_rng(2000)
            r, c = rng.integers(0, n, 4096), rng.integers(0, n, 4096)
            cf = p.closed_form_entries(xh, r, c)
            row["closed_form_max_err_over_max_entry"] = float(np.max(np.abs(Hd[r, c] - cf)) / np.max(np.abs(cf)))
        res[f"n{n}"] = row
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
