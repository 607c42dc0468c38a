#!/usr/bin/env python
"""c2_step_ledger.py — where the time of one C2 step goes, on the GPU.

Two measurements, printed as markdown tables:

1. Kernel ledger.  The C2 problem exactly as bench.py builds it (N = 10^7 tridiagonal, 3 cyclic colours, CSC J), one
   torch.profiler trace of `--steps` Jacobian calls launched eagerly and one of the same calls replayed from the captured
   CUDA graph.  For every kernel of a step, in issue order: its mean duration and the mean gap before it, measured from
   the trace timestamps as its start minus the latest end of any kernel that started before it (negative: it started
   while an earlier kernel was still running — a side stream, or a programmatic dependent launch).  Below each table the
   step period, the time some kernel was running (union of the kernel intervals) and the rest, when none was.

2. Stream ceilings.  Three pure streams at C2 sizes (n = 10^7 doubles per vector), timed with CUDA events: read-only,
   1 read : 3 writes (the perturbation's mix) and 4 reads : 3 writes (the forward scatter's mix), each at a few grid
   sizes, best kept.  They give a measured ceiling for each kernel's traffic mix on this card.

The card's name and power limit are read in the same run and printed with the numbers.  Needs a GPU; without one it
exits with status 2.  Traces are written under --out (default: a temporary directory).

    python scripts/c2_step_ledger.py [--fdtype forward|central] [--steps 20] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def short(name):
    name = name.replace("void ", "").replace("fdb::", "").replace("(anonymous namespace)::", "")
    depth, out = 0, []
    for ch in name:                       # drop the argument list, keep the template arguments
        if ch == "(" and depth == 0:
            break
        depth += ch == "<"
        depth -= ch == ">"
        out.append(ch)
    s = "".join(out)
    return s if len(s) <= 90 else s[:87] + "..."


def kernels_of(trace_path):
    ev = json.loads(Path(trace_path).read_text())["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel" and "dur" in e]
    ks.sort(key=lambda e: float(e["ts"]))
    return [(float(e["ts"]), float(e["dur"]), short(e["name"]), e.get("args", {}).get("stream")) for e in ks]


def ledger(ks, steps, title, bytes_of):
    if not ks or len(ks) % steps:
        print(f"\n{title}: {len(ks)} kernels in {steps} steps: not a whole number per step, no table")
        return
    per = len(ks) // steps
    rows = [ks[i * per:(i + 1) * per] for i in range(steps)]
    ends, prev_end = [], None
    gaps = [[] for _ in range(per)]
    for r in rows:
        for j, (ts, dur, _, _) in enumerate(r):
            if prev_end is not None:
                gaps[j].append(ts - prev_end)
            prev_end = ts + dur if prev_end is None else max(prev_end, ts + dur)
        ends.append(prev_end)
    print(f"\n{title}\n")
    print("| # | stream | kernel | mean duration (µs) | mean gap before (µs) | GB/s |")
    print("|---|---|---|---|---|---|")
    for j in range(per):
        d = statistics.mean(r[j][1] for r in rows)
        g = statistics.mean(gaps[j]) if gaps[j] else float("nan")
        b = bytes_of(rows[0][j][2])
        rate = f"{b / (d * 1e-6) / 1e9:.0f}" if b else ""
        print(f"| {j} | {rows[0][j][3]} | `{rows[0][j][2]}` | {d:.1f} | {g:+.1f} | {rate} |")
    period = statistics.mean(rows[i + 1][0][0] - rows[i][0][0] for i in range(steps - 1))
    busy = []
    for r in rows[:-1]:
        iv = sorted((ts, ts + dur) for ts, dur, _, _ in r)
        tot, cs, ce = 0.0, iv[0][0], iv[0][1]
        for a, b in iv[1:]:
            if a > ce:
                tot += ce - cs
                cs, ce = a, b
            else:
                ce = max(ce, b)
        busy.append(tot + ce - cs)
    bu = statistics.mean(busy)
    print(f"\nstep period {period:.1f} µs; some kernel running {bu:.1f} µs; no kernel running {period - bu:.1f} µs")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--fdtype", default="forward", choices=["forward", "central"])
    ap.add_argument("--steps", type=int, default=20, help="Jacobian calls per trace")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a temporary directory)")
    ap.add_argument("--no-probes", dest="probes", action="store_false", help="skip the stream ceilings")
    args = ap.parse_args()
    if args.steps < 2:
        ap.error("--steps must be at least 2")

    import torch
    if not torch.cuda.is_available():
        print("c2_step_ledger: no CUDA device — this script measures the GPU and has nothing to do without one",
              file=sys.stderr)
        sys.exit(2)
    import bench
    import _bootstrap
    from torch.profiler import ProfilerActivity, profile
    pkg = _bootstrap.load_package()
    dev = torch.device("cuda:0")
    out = Path(args.out) if args.out else Path(tempfile.mkdtemp(prefix="c2_ledger_"))
    out.mkdir(parents=True, exist_ok=True)
    print(f"card: {card()}")
    print(f"C2 {args.fdtype}, N = 10^7, {args.steps} steps per trace; traces under {out}")

    n = 10_000_000
    NP = 3
    ctrl = 2 if args.fdtype == "central" else 1

    for use_graph in (False, True):
        prob = bench.build_gpu_problem(pkg, "c2", args.fdtype, dev, 0, 1, 1, use_graph=use_graph)
        J, f, x, cache = prob["J"], prob["f"], prob["x"], prob["cache"]

        def step():
            pkg.finite_difference_jacobian_(J, f, x, cache)

        for _ in range(max(args.warmup, 3)):
            step()
        torch.cuda.synchronize()
        info = cache._last_plan.info()
        scat_bytes = info["moved_bytes_scatter"]

        def bytes_of(name):
            if name.startswith("perturb_colors"):
                return 8 * n + 8 * n * NP * ctrl
            if name.startswith("diff_scatter_staged"):
                return scat_bytes
            if name.startswith("color_sumsq"):
                return 8 * n
            if "tridiag" in name:
                return 16 * n
            return 0

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
        tag = "graph" if use_graph else "eager"
        path = out / f"c2_{args.fdtype}_{tag}.pt.trace.json"
        prof.export_chrome_trace(str(path))
        ledger(kernels_of(path), args.steps, f"C2 {args.fdtype}, {tag} launches", bytes_of)
        del prob, J, f, x, cache
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    if not args.probes:
        return
    synth = pkg._lib.synth()
    src = torch.ones(4 * n, dtype=torch.float64, device=dev)
    dst = torch.empty(3 * n, dtype=torch.float64, device=dev)
    sink = torch.zeros(1, dtype=torch.float64, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream
    print("\nStream ceilings (n = 10^7 doubles per vector, 16-byte streaming accesses, CUDA events, best grid)\n")
    print("| mix | bytes | best time (µs) | GB/s | grid |")
    print("|---|---|---|---|---|")
    for reads, writes, label in ((1, 0, "read-only"), (1, 3, "1 read : 3 writes (perturbation)"),
                                 (4, 3, "4 reads : 3 writes (forward scatter)")):
        best = None
        for blocks in (sms * 8, sms * 32, sms * 128):
            def launch():
                rc = synth.fdbs_stream_probe(src.data_ptr(), n, reads, dst.data_ptr(), n, writes, n, blocks,
                                             sink.data_ptr(), stream)
                if rc:
                    raise RuntimeError(f"fdbs_stream_probe returned {rc}")
            for _ in range(3):
                launch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 50
            e0.record()
            for _ in range(reps):
                launch()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / reps
            if best is None or us < best[0]:
                best = (us, blocks)
        nbytes = (reads + writes) * n * 8
        print(f"| {label} | {nbytes / 1e6:.0f} MB | {best[0]:.1f} | {nbytes / (best[0] * 1e-6) / 1e9:.0f} | {best[1]} |")


if __name__ == "__main__":
    main()
