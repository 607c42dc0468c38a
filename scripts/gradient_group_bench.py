"""Multi-GPU gradients (distributed.GroupGradient): time per gradient of the single plan and of groups over repeated and
distinct devices, with every group's df bit-compared with the single plan's.

    python scripts/gradient_group_bench.py [--out FILE]

f is the synthetic quartic of include/fdjac_synth.h (fdbs_quartic), max_batch 4096, n = 10^4 and 10^5, forward and
central.  Arms: the single plan (finite_difference_gradient_); group [0]; group [0, 0] (two members on one card: the
group's overhead, not scaling); and, when k > 1 GPUs are visible, group [0 .. k-1].  Each arm is warmed up, then timed
with CUDA events on the root stream over enough calls to exceed one second, in three rounds that alternate the arms;
gradient_s is the best round.  Prints one JSON line; the card's name, power limit and max SM clock are read in the same
run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import subprocess
import sys
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


class Problem:
    def __init__(self, pkg, n, seed=7):
        rng = np.random.default_rng(seed + n)
        self.pkg, self.n, self.a, self.w = pkg, n, 0.5 + rng.random(n), rng.random(n) * 2 - 1
        self.x = torch.empty(n, dtype=torch.float64, device="cuda:0")
        pkg._lib.synth().fdbs_fill_x(self.x.data_ptr(), n, 0xC0FFEE + n, None)
        self._keep = []

    def fn(self, d):
        dev = torch.device("cuda", d)
        da, dw = torch.from_numpy(self.a).to(dev), torch.from_numpy(self.w).to(dev)
        ctx = self.pkg._lib.ScalarCtx(self.n, da.data_ptr(), dw.data_ptr(), 0)
        self._keep.append((da, dw, ctx))
        return self.pkg.NativeFn(C.cast(self.pkg._lib.synth().fdbs_quartic, C.c_void_p).value, ctx)


def timed(call, min_s=1.0):
    """(seconds per call, calls): one warm-up call, one call to size the window, then >= min_s of calls between two
    events on the current (root) stream"""
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
    return e0.elapsed_time(e1) / 1e3 / reps, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gradient_group_bench needs a GPU"
    pkg = _bootstrap.load_package()
    from finitediff_jl_b200 import distributed
    k = torch.cuda.device_count()
    res = {"metric": "gradient_group", "card": card(), "visible_gpus": k, "f": "fdbs_quartic", "max_batch": 4096}
    arms = [[0], [0, 0]] + ([list(range(k))] if k > 1 else [])
    rounds = 3
    res["rounds"] = rounds
    for n in (10_000, 100_000):
        p = Problem(pkg, n)
        for fdtype in ("forward", "central"):
            df1 = torch.empty(n, dtype=torch.float64, device="cuda:0")
            cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device="cuda:0"), p.x, fdtype, max_batch=4096)
            f0 = p.fn(0)
            calls = {"single": lambda df1=df1, f0=f0, cache=cache: pkg.finite_difference_gradient_(df1, f0, p.x, cache)}
            groups, outs = {}, {}
            for devices in arms:
                name = "group_" + "_".join(map(str, devices))
                g = distributed.GroupGradient(n, devices, fdtype, max_batch=4096)
                fs = [p.fn(d) for d in devices]
                df = torch.empty(n, dtype=torch.float64, device="cuda:0")
                groups[name], outs[name] = g, df
                calls[name] = (lambda g=g, fs=fs, df=df: g.run(fs, p.x, df))
            # the arms alternate round by round, so that clock and neighbour drift fall on all of them alike
            times = {name: [] for name in calls}
            for _ in range(rounds):
                for name, call in calls.items():
                    t, reps = timed(call)
                    times[name].append(t)
            ref = df1.cpu().numpy().view(np.uint64)
            best = {name: min(v) for name, v in times.items()}
            row = {"single": {"gradient_s": best["single"], "rounds_s": times["single"]}}
            for name, g in groups.items():
                got = outs[name].cpu().numpy().view(np.uint64)
                row[name] = {
                    "gradient_s": best[name], "rounds_s": times[name], "speedup_vs_single": best["single"] / best[name],
                    "member_columns": [e - b for b, e in (pl.dense_range() for pl in g.plans)],
                    "bit_identical_to_single": bool(np.array_equal(got, ref)),
                    "entries_differing": int(np.count_nonzero(got != ref))}
                g.close()
            res[f"n{n}_{fdtype}"] = row
            del cache
            torch.cuda.empty_cache()
    res["scaling"] = "measured" if k > 1 else "not measured: one GPU visible ([0, 0] measures the group's overhead)"
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
