"""Derivatives with a scalar input per step size on the device (fdb_derivative): kernel times of deriv_points and
deriv_quotient against the measured streaming ceiling of their read:write mix, and bit parity with the CPU restatement.

    python scripts/derivative_bench.py [--n N] [--reps R] [--out FILE]

Workloads: the elementwise derivative (finite_difference_derivative!, src/derivatives.jl:197-233) at n = 10^8 in forward,
central and complex mode, and the scalar -> vector gradient (finite_difference_gradient! at a number, src/gradients.jl:
477-533) at m = 10^8, with the cheap native synthetic f of include/fdjac_synth.h (fdbs_poly / fdbs_tpoly, complex twins).

Kernel times come from CUDA events: the timed f (a ctypes wrapper around the native f) records an event when it is first
called, which ends the points pass, and another after its last launch, which starts the quotient pass; an event after the
call ends it.  A device sleep before each call keeps the host ahead of the GPU, so no event waits for a launch.  The
ceilings are fdbs_stream_probe at the same read:write mix, in the same run: 1:1 (forward points), 1:2 (central points;
complex points, 8 B read and 16 B written per component), 3:1 (forward / central quotient), 2:1 (complex quotient; scalar
gradient quotient).  Parity: a 10^6-element slice of df bit-compared with the restatement.  Prints one JSON line; the
card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import _bootstrap  # noqa: E402
from scalar_oracle import fd_scalar_oracle as so  # noqa: E402

# compulsory bytes per component (derivative) or per output (gradient) of each pass, and the probe mix it streams
PASSES = {
    "forward": ((16, (1, 1)), (32, (3, 1))),
    "central": ((24, (1, 2)), (32, (3, 1))),
    "complex": ((24, (1, 2)), (24, (2, 1))),
}
GRAD_QUOTIENT = (24, (2, 1))
SLEEP_CYCLES = 2_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def probe_ceilings(pkg, n, reps):
    """GB/s of fdbs_stream_probe for each mix: best over a few grid sizes."""
    S = pkg._lib.synth()
    src = torch.empty(3 * n + 8, dtype=torch.float64, device="cuda").uniform_()
    dst = torch.empty(2 * n + 8, dtype=torch.float64, device="cuda")
    sink = torch.zeros(1, dtype=torch.float64, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {}
    for r, w in sorted({m for p in PASSES.values() for _, m in p} | {GRAD_QUOTIENT[1]}):
        best = 0.0
        for blocks in (sms * 4, sms * 8, sms * 16):
            run = lambda: S.fdbs_stream_probe(src.data_ptr(), n, r, dst.data_ptr(), n, w, n, blocks, sink.data_ptr(), None)
            assert run() == 0
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            best = max(best, 8.0 * n * (r + w) * reps / (e0.elapsed_time(e1) * 1e-3) / 1e9)
        out[f"{r}:{w}"] = best
    return out


class TimedFn:
    """ctypes fdb_fn that calls a native synthetic f and records the pass boundaries on the call's stream."""

    def __init__(self, native, ctx, calls_per_derivative):
        self.native, self.ctx, self.per = native, ctx, calls_per_derivative
        self.k = 0
        self.marks = []
        self.cf = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                              C.c_void_p)(self._call)
        self.address = C.cast(self.cf, C.c_void_p).value

    def _call(self, _ctx, fx, x, batch, ldfx, ldx, stream):
        s = torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream()
        if self.k % self.per == 0:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(s)
            self.marks.append(ev)
        rc = self.native(C.cast(C.pointer(self.ctx), C.c_void_p), fx, x, batch, ldfx, ldx, stream)
        self.k += 1
        if self.k % self.per == 0:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(s)
            self.marks.append(ev)
        return rc


def time_calls(call, tf, reps):
    """(points ms, quotient ms) per call, median over reps."""
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    tf.marks.clear()
    starts, ends = [], []
    for _ in range(reps):
        torch.cuda._sleep(SLEEP_CYCLES)
        e0, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e3.record()
        starts.append(e0)
        ends.append(e3)
    torch.cuda.synchronize()
    pts = [s.elapsed_time(tf.marks[2 * i]) for i, s in enumerate(starts)]
    quo = [tf.marks[2 * i + 1].elapsed_time(e) for i, e in enumerate(ends)]
    return float(np.median(pts)), float(np.median(quo))


def coefficients(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = 0.5 + torch.rand(n, dtype=torch.float64, device="cuda", generator=g)
    w = torch.rand(n, dtype=torch.float64, device="cuda", generator=g) * 2 - 1
    return a, w


def bench_derivative(pkg, mode, n, reps, ceil, sample):
    L = pkg._lib
    a, w = coefficients(n, 1)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0xD311 + n, None)
    ctx = L.ScalarCtx(n, a.data_ptr(), w.data_ptr(), 0)
    native = getattr(L.synth(), "fdbs_poly_c" if mode == "complex" else "fdbs_poly")
    tf = TimedFn(native, ctx, 1 if mode == "complex" else 2)
    fn = pkg.NativeFn(tf.address, None)
    cache = pkg.DerivativeCache(x, None, None, mode)
    df = torch.empty(n, dtype=torch.float64, device="cuda")
    pts_ms, quo_ms = time_calls(lambda: pkg.finite_difference_derivative_(df, fn, x, cache), tf, reps)
    # parity on a sampled slice: component i depends on x[i], a[i], w[i] only
    lo = (n // 2) // 1024 * 1024 + 3
    sl = slice(lo, min(n, lo + sample))
    twin = so.SynthScalar(sl.stop - sl.start, a[sl].cpu().numpy(), w[sl].cpu().numpy())
    ref = so.derivative(twin.native("synth_poly_c" if mode == "complex" else "synth_poly"), x[sl].cpu().numpy(),
                        {"forward": so.FORWARD, "central": so.CENTRAL, "complex": so.COMPLEX}[mode])
    got = df[sl].cpu().numpy()
    parity = bool(np.array_equal(got.view(np.uint64), ref["df"].view(np.uint64)))
    (pb, pmix), (qb, qmix) = PASSES[mode]
    info = cache._last_plan.info()
    assert info["alg_bytes_scatter"] == (pb + qb) * n
    return {
        "n": n, "parity_slice": [sl.start, sl.stop], "bit_identical": parity,
        "points": _row(pts_ms, pb * n, pmix, ceil), "quotient": _row(quo_ms, qb * n, qmix, ceil),
    }


def bench_scalar_gradient(pkg, m, reps, ceil, sample):
    L = pkg._lib
    a, w = coefficients(m, 2)
    ctx = L.ScalarCtx(m, a.data_ptr(), w.data_ptr(), 0)
    tf = TimedFn(L.synth().fdbs_tpoly, ctx, 2)
    fn = pkg.NativeFn(tf.address, None)
    df = torch.empty(m, dtype=torch.float64, device="cuda")
    t = torch.tensor([0.7318], dtype=torch.float64, device="cuda")
    cache = pkg.GradientCache(df, 0.0, "central")
    pts_ms, quo_ms = time_calls(lambda: pkg.finite_difference_gradient_(df, fn, t, cache), tf, reps)
    sl = slice(m // 3, min(m, m // 3 + sample))
    twin = so.SynthScalar(sl.stop - sl.start, a[sl].cpu().numpy(), w[sl].cpu().numpy())
    ref = so.scalar_gradient(twin.native("synth_tpoly"), 0.7318, sl.stop - sl.start, so.CENTRAL)
    parity = bool(np.array_equal(df[sl].cpu().numpy().view(np.uint64), ref["df"].view(np.uint64)))
    qb, qmix = GRAD_QUOTIENT
    return {"m": m, "mode": "central", "parity_slice": [sl.start, sl.stop], "bit_identical": parity,
            "points_ms": pts_ms, "quotient": _row(quo_ms, qb * m, qmix, ceil)}


def _row(ms, nbytes, mix, ceil):
    gbs = nbytes / (ms * 1e-3) / 1e9
    c = ceil[f"{mix[0]}:{mix[1]}"]
    return {"ms": round(ms, 4), "bytes": nbytes, "GBps": round(gbs, 1), "mix": f"{mix[0]}:{mix[1]}",
            "ceiling_GBps": round(c, 1), "share_of_ceiling": round(gbs / c, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--sample", type=int, default=1_000_000)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("derivative_bench.py measures the device path and needs a GPU")
    pkg = _bootstrap.load_package()
    so.build()
    ceil = probe_ceilings(pkg, a.n, max(20, a.reps // 10))
    res = {"card": card(), "probe_ceilings_GBps": {k: round(v, 1) for k, v in ceil.items()}}
    for mode in ("forward", "central", "complex"):
        res[f"derivative_{mode}"] = bench_derivative(pkg, mode, a.n, a.reps, ceil, a.sample)
        torch.cuda.empty_cache()
    res["scalar_gradient_central"] = bench_scalar_gradient(pkg, a.n, a.reps, ceil, a.sample)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
