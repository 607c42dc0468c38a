"""GPU parity of the colour step sizes at the ends of the fp64 range (run with -m gpu on an H100).

The reference's norm(x2) (jacobians.jl:560) is OpenBLAS dnrm2 for n >= 32, an x87 80-bit sum without overflow or
underflow for any double, and stdlib generic_norm2 for n < 32, which rescales only when maxabs^2 == 0 or n*maxabs^2
overflows.  A plain fp64 sum of squares gives Inf for |x| >~ 1.34e154, 0 when every square underflows, and a value
up to 1e-11 off when the squares are subnormal but their sum is not.  Every case puts colour 2 at such an extreme and
keeps the other colours in range, then holds the bars of the other GPU parity tests: every f! argument and J bit for
bit against the oracle fed the device step sizes, and the device step sizes within rtol 1e-13 of the oracle's own (Inf
and NaN where the oracle's are).  Guards against vacuous passes: the oracle's own step size of colour 2 is finite, Inf
or NaN as each case states, and J has no NaN where the oracle's own J has none.  The kernels a call ran are read from a
torch.profiler trace, so each input provably reaches the step-size path it is meant for; the traces are taken in a child
process (python tests/test_gpu_eps_range.py --trace-paths), because hundreds of profiler sessions in the pytest process
make later traces in it (tests/test_gpu_multiwave.py) miss kernels."""
import json
import os
import re
import subprocess
import sys
import tempfile
from fractions import Fraction

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

from _util import assert_same_bits, cyc_colors, fdb_env, tridiag_csc, tridiagonal_coo  # noqa: E402

FD = {"forward": 0, "central": 1}
MODES = [("forward", 1.0), ("forward", -1.0), ("central", 1.0)]
TRAP = 4.79825341824841e-157     # its square is subnormal and rounded by nearly half an ulp (test_trap_value)
T = 2.0 ** -900                  # the device rescues sums of squares below this (n >= 32)


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))


# f! = the tridiagonal stencil scaled by 1/4 before the sums: finite for every finite x (case "norm_inf" sits at 1e308)
def f_np(dx, x):
    n = len(x)
    dx[1:n - 1] = (x[0:n - 2] * 0.25 - x[1:n - 1] * 0.5) + x[2:n] * 0.25
    dx[0] = x[0] * -0.5 + x[1] * 0.25
    dx[n - 1] = x[n - 2] * 0.25 - x[n - 1] * 0.5


def f_t(dx, x):
    n = x.shape[-1]
    dx[..., 1:n - 1] = (x[..., 0:n - 2] * 0.25 - x[..., 1:n - 1] * 0.5) + x[..., 2:n] * 0.25
    dx[..., 0] = x[..., 0] * -0.5 + x[..., 1] * 0.25
    dx[..., n - 1] = x[..., n - 2] * 0.25 - x[..., n - 1] * 0.5


def recording_t(log):
    def f(dx, x):
        log.extend(np.array(r, copy=True) for r in x.reshape(-1, x.shape[-1]).cpu().numpy())
        f_t(dx, x)
    f.batched = False
    return f


def recording_np(log):
    def f(dx, x):
        log.append(np.array(x, copy=True))
        f_np(dx, x)
    return f


def traced(fn):
    """Run fn() under torch.profiler (CUDA activity); return the names of the kernels it launched, in order."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # kernel records at either end of a session can be missing from its trace: the first few once the profiler has
        # sat idle for a minute or so in a process, the last one when the session stops right after it (seen for the
        # staged scatter, the last launch of a forward call).  Throwaway launches take those places on both sides.
        pad = torch.empty(1, device="cuda")
        for _ in range(64):
            pad.fill_(0.0)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        for _ in range(64):
            pad.fill_(0.0)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            events = json.load(fh)["traceEvents"]
    return [e["name"] for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))]


def count(kernels, name):
    return sum(1 for k in kernels if re.search(r"\b" + name + r"[<(]", k))


# ------------------------------------------------------------------------------------------------------------- inputs
# name -> (absstep, what the oracle's own step size of colour 2 is: "finite" | "inf" | "nan")
CASES = {
    "sq_overflow": (None, "finite"),     # A: |x| in 10^[155, 300]: squares overflow, the norm does not
    "norm_inf": (None, "inf"),           # B: components near 1e308, enough of them that the norm overflows
    "sq_zero": (0.0, "finite"),          # C: |x| in 10^[-320, -163], 5e-324 and signed zeros: squares underflow to 0
    "trap": (0.0, "finite"),             # D: subnormal squares, each rounded, whose sum is a normal number
    "below_T": (0.0, "finite"),          # D: a sum of squares just below the rescue threshold 2^-900 ...
    "above_T": (0.0, "finite"),          #    ... and just above it
    "partly_sub": (0.0, "finite"),       # E: |x| in 10^[-160, -150]: some squares subnormal
    "mixed": (None, "finite"),           # F: 1e200 and 1e-200 in one colour
    "inf_in_big": (None, "inf"),         # G: +Inf inside a colour whose squares overflow
    "nan_with_big": (None, "nan"),       # G: NaN together with 1e200
}


def colour_values(kind, m, rng):
    """m values for colour 2's components."""
    sign = np.where(rng.random(m) < 0.5, -1.0, 1.0)
    if kind == "sq_overflow":
        return sign * 10.0 ** rng.uniform(155, 300, m)
    if kind == "norm_inf":
        assert m >= 4                        # sqrt(m) * 0.9e308 > DBL_MAX
        return sign * rng.uniform(0.9e308, 1.1e308, m)
    if kind == "sq_zero":
        v = sign * 10.0 ** rng.uniform(-320, -163, m)
        v[: min(m, 6)] = [5e-324, -5e-324, 0.0, -0.0, 1e-323, -0.0][: min(m, 6)]
        return v
    if kind == "trap":
        assert m * TRAP * TRAP > 2.2250738585072014e-308        # the plain sum is a normal number
        return np.full(m, TRAP)
    if kind in ("below_T", "above_T"):
        v = np.sqrt(T / m) * (1 - 1e-6 if kind == "below_T" else 1 + 1e-6)
        s = float(np.sum(np.full(m, v) ** 2))
        assert (s < T) == (kind == "below_T")
        return np.full(m, v) * sign
    if kind == "partly_sub":
        return sign * 10.0 ** rng.uniform(-160, -150, m)
    if kind == "mixed":
        return np.where(np.arange(m) % 2 == 0, 1e200, 1e-200) * sign
    if kind == "inf_in_big":
        v = sign * 1e200
        v[m // 2] = np.inf
        return v
    if kind == "nan_with_big":
        v = sign * 1e200
        v[m // 2] = np.nan
        return v
    if kind == "in_range":
        return sign * rng.uniform(0.5, 2.0, m)
    raise ValueError(kind)


def make_x(kind, cv, seed=5):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.5, 2.0, len(cv)) * np.where(rng.random(len(cv)) < 0.5, -1.0, 1.0)
    c2 = np.flatnonzero(cv == 2)
    x[c2] = colour_values(kind, len(c2), rng)
    return x


def table_colors(N, C):
    """A valid distance-2 colouring of the tridiagonal pattern that the plan cannot take as cyclic: C colours in the
    order 2, 3, .., C, 1, repeated."""
    return (np.arange(N) + 1) % C + 1


def trap_colors(N, C):
    """A valid distance-2 colouring of the tridiagonal pattern with colour 2 on every third column (N/3 components:
    enough for the "trap" sum to be a normal number) and the other C - 1 colours cycling over the rest; cyclic for C = 3."""
    cv = np.empty(N, dtype=np.int64)
    rest = np.flatnonzero(np.arange(N) % 3 != 1)
    cv[np.arange(N) % 3 == 1] = 2
    cv[rest] = np.array([1] + list(range(3, C + 1)))[np.arange(len(rest)) % (C - 1)]
    return cv


def colours(case, N, C, colouring="cyclic"):
    if case == "trap":
        return trap_colors(N, C)
    return cyc_colors(N, C) if colouring == "cyclic" else table_colors(N, C)


# ---------------------------------------------------------------------------------------------------------- harness
def problem(pkg, oracle, dev, form, N):
    """(J on the device, its value tensor, the oracle's Problem or None without an oracle, the oracle's J length)"""
    if form == "csc":
        colptr, rowval = tridiag_csc(N)
        J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval),
                                torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
        return J, J.nzval, oracle and oracle.Problem.csc_same(N, N, colptr, rowval), len(rowval)
    if form == "banded":
        J = pkg.BandedMatrix(N, N, 1, 1, device=dev)
        J.data.fill_(float("nan"))
        return J, J.data, oracle and oracle.Problem.banded(N, N, 1, 1), 3 * N
    if form == "coo":                        # Tridiagonal: structural entries with slots into [dl; d; du]
        J = pkg.Tridiagonal(N, device=dev)
        J.buf.fill_(float("nan"))
        rows, cols, slots = tridiagonal_coo(N)
        return J, J.buf, oracle and oracle.Problem.coo_to_slots(N, N, rows, cols, slots, 3 * N - 2), 3 * N - 2
    raise ValueError(form)


def run(pkg, oracle, dev, x_np, fdtype, cv, *, form="csc", dir=1.0, absstep=None, env=None, unaligned=False,
        colour2=None):
    """One Jacobian on the device and in the oracle; asserts the parity bars and returns the device step sizes.
    colour2: "finite" | "inf" | "nan", what the oracle's own step size of colour 2 must be."""
    N = len(x_np)
    xbuf = torch.zeros(N + 1, dtype=torch.float64, device=dev)
    x = xbuf[1:] if unaligned else xbuf[:N]
    x.copy_(torch.from_numpy(x_np))
    J, jv, P, jlen = problem(pkg, oracle, dev, form, N)
    log = []
    kw = {} if absstep is None else {"absstep": absstep}
    with fdb_env(**(env or {})):
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
        pkg.finite_difference_jacobian_(J, recording_t(log), x, cache, dir=dir, **kw)
    torch.cuda.synchronize()
    assert_same_bits(x, x_np, "the caller's x is never written")
    eps = cache._last_plan.eps()
    got = jv.cpu().numpy()
    olog = []
    ref = np.full(jlen, np.nan)
    r = oracle.jacobian(P, ref, recording_np(olog), x_np.copy(), fdtype=FD[fdtype], colorvec=cv, eps_override=eps,
                        dir=dir, **kw)
    own_J = np.full(jlen, np.nan)
    own = oracle.jacobian(P, own_J, f_np, x_np.copy(), fdtype=FD[fdtype], colorvec=cv, dir=dir, **kw)
    what = f"{form} {fdtype} dir={dir} env={env} unaligned={unaligned}"
    assert len(log) == len(olog) == r["fcalls"], what
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a, b, f"{what}: argument of f! call {i}")
    assert_same_bits(got, ref, f"{what}: J")
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13, atol=0, err_msg=what)
    # vacuous-pass guards
    if colour2 is not None:
        e2 = own["eps"][1]
        assert {"finite": np.isfinite(e2), "inf": np.isinf(e2), "nan": np.isnan(e2)}[colour2], (what, e2)
    assert np.isfinite(np.delete(own["eps"], 1)).all()
    assert not np.isnan(got[~np.isnan(own_J)]).any(), f"{what}: NaN in J where the oracle's own J has none"
    return eps


def test_trap_value():
    # the square of TRAP is subnormal and off by nearly half of the subnormal spacing 2^-1074
    sq = TRAP * TRAP
    assert 0 < sq < 2.2250738585072014e-308
    off = abs(Fraction(sq) - Fraction(TRAP) ** 2) / Fraction(2) ** -1074
    assert Fraction(45, 100) < off <= Fraction(1, 2)


# ------------------------------------------------------------------------ which step-size path each input reaches
# (name, form, C, N, switches, {kernel: launches}) — the configurations of the parity tests below
TRACE_PATHS = [
    ("reg_cyclic", "csc", 3, 20_011, {}, {"color_sumsq_reg": 1}),
    ("reg_table_banded", "banded", 7, 20_011, {"SM_COUNT": 1}, {"color_sumsq_reg": 1}),
    ("lists", "csc", 20, 30_011, {}, {"color_sumsq_lists": 1, "finalize_eps_lists": 1}),
    ("win_banded", "banded", 10, 20_011, {}, {"color_sumsq_win": 1, "finalize_eps": 1}),
    ("win_coo", "coo", 10, 20_011, {}, {"color_sumsq_win": 1, "finalize_eps": 1}),
    ("win_csc_no_lists", "csc", 20, 20_011, {"NO_EPS_LISTS": 1}, {"color_sumsq_win": 1, "finalize_eps": 1}),
    ("two_windows", "csc", 600, 600 * 40 + 7, {"NO_EPS_LISTS": 1}, {"color_sumsq_win": 2, "finalize_eps": 2}),
    ("reg_n13", "csc", 3, 13, {}, {"color_sumsq_reg": 1}),
    ("lists_n13", "csc", 10, 13, {}, {"color_sumsq_lists": 1, "finalize_eps_lists": 1}),
    ("win_n13", "csc", 10, 13, {"NO_EPS_LISTS": 1}, {"color_sumsq_win": 1, "finalize_eps": 1}),
]


def _trace_paths():
    """Child process: one traced forward Jacobian per (path, input); prints {"path/input": [kernel names]} as JSON."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import _bootstrap
    pkg = _bootstrap.load_package()
    dev = torch.device("cuda:0")
    out = {}
    for name, form, C, N, env, _ in TRACE_PATHS:
        for case in CASES:
            if (N < 32 and case != "sq_overflow") or (name == "two_windows" and case == "trap"):
                continue
            n = 300_007 if case == "trap" else N
            cv = colours(case, n, C, "table" if "table" in name else "cyclic") if N > 32 else cyc_colors(n, C)
            x = torch.from_numpy(make_x(case, cv) if N > 32 else np.full(n, 1e300)).to(dev)
            J, _, _, _ = problem(pkg, None, dev, form, n)
            absstep = CASES[case][0]
            with fdb_env(**env):
                cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J)
                out[f"{name}/{case}"] = traced(lambda: pkg.finite_difference_jacobian_(
                    J, lambda dx, xx: f_t(dx, xx), x, cache, **({} if absstep is None else {"absstep": absstep})))
    x = torch.from_numpy(np.array([1.7e308, 5e-324, 1.0] * 100)).to(dev)
    J = pkg.zeros_colmajor(300, 300, dev)
    cache = pkg.JacobianCache(x, torch.zeros(300, dtype=torch.float64, device=dev), "forward")
    out["dense/extremes"] = traced(lambda: pkg.finite_difference_jacobian_(J, lambda dx, xx: f_t(dx, xx), x, cache,
                                                                           absstep=0.0))
    print(json.dumps(out))


def test_every_input_reaches_its_path(pkg):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--trace-paths"], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for name, _, _, N, _, want in TRACE_PATHS:
        for case in (CASES if N > 32 else ["sq_overflow"]):
            if name == "two_windows" and case == "trap":
                continue
            ks = got[f"{name}/{case}"]
            for kernel, launches in want.items():
                assert count(ks, kernel) == launches, (name, case, kernel, ks)
    assert count(got["dense/extremes"], "component_eps"), got["dense/extremes"]


# ------------------------------------------------------------------------------ color_sumsq_reg (C <= 8): every input


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("form", ["csc", "banded"])
@pytest.mark.parametrize("C,colouring", [(3, "cyclic"), (7, "table")])
@pytest.mark.parametrize("fdtype,dir", MODES)
def test_register_path(pkg, oracle, dev, case, form, C, colouring, fdtype, dir):
    N = 300_007 if case == "trap" else 20_011
    cv = colours(case, N, C, colouring)
    absstep, c2 = CASES[case]
    run(pkg, oracle, dev, make_x(case, cv), fdtype, cv, form=form, dir=dir, absstep=absstep, colour2=c2)


@pytest.mark.parametrize("case", ["sq_overflow", "norm_inf", "sq_zero", "trap", "partly_sub", "mixed"])
def test_register_path_geometry(pkg, oracle, dev, case):
    # x only 8-byte aligned (scalar loads), one or two tiles in flight, 1 and 3 "SMs": the same step-size bits
    N = 300_007 if case == "trap" else 20_011
    absstep, c2 = CASES[case]
    for C in (3, 7):
        cv = colours(case, N, C)
        x = make_x(case, cv)
        runs = []
        for unaligned in (False, True):
            for env in ({}, {"EPS_DEPTH": 1}, {"SM_COUNT": 1}, {"SM_COUNT": 3}):
                runs.append(run(pkg, oracle, dev, x, "forward", cv, absstep=absstep, env=env, unaligned=unaligned,
                                colour2=c2))
        # EPS_DEPTH keeps the summation order: the same bits.  Other grids (SM_COUNT) reorder the in-range sums; the
        # rescued colour 2 depends neither on the grid nor on the alignment of x.
        assert_same_bits(runs[1], runs[0], f"C={C}: EPS_DEPTH=1")
        assert_same_bits(runs[5], runs[4], f"C={C}: EPS_DEPTH=1, x unaligned")
        for r in runs:
            assert_same_bits(r[1], runs[0][1], f"C={C}: colour 2 at every grid")


# ------------------------------------------------- color_sumsq_lists + finalize_eps_lists (C > 8, CSC): every input
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("fdtype,dir", MODES)
def test_list_path(pkg, oracle, dev, case, fdtype, dir):
    N = 300_007 if case == "trap" else 30_011
    cv = colours(case, N, 20)
    x = make_x(case, cv)
    absstep, c2 = CASES[case]
    runs = [run(pkg, oracle, dev, x, fdtype, cv, dir=dir, absstep=absstep, env=env, colour2=c2)
            for env in ({}, {"SM_COUNT": 1}, {"SM_COUNT": 3})]
    for r in runs[1:]:
        assert_same_bits(r, runs[0], "the list path does not depend on the grid")


# --------------------------------------------------------------------- color_sumsq_win + finalize_eps: every input
WIN = [  # (name, form, C, env)
    ("banded", "banded", 10, {}),
    ("coo", "coo", 10, {}),
    ("csc_no_lists", "csc", 20, {"NO_EPS_LISTS": 1}),
    ("two_windows", "csc", 600, {"NO_EPS_LISTS": 1}),
]


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("path", [w[0] for w in WIN])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_window_path(pkg, oracle, dev, case, path, fdtype):
    _, form, C, env = next(w for w in WIN if w[0] == path)
    if path == "two_windows":
        if case == "trap":
            pytest.skip("600 colours leave colour 2 too few components for a normal sum of subnormal squares")
        N = 600 * 40 + 7
    else:
        N = 300_007 if case == "trap" else 20_011
    cv = colours(case, N, C)
    absstep, c2 = CASES[case]
    run(pkg, oracle, dev, make_x(case, cv), fdtype, cv, form=form, absstep=absstep, env=env, colour2=c2)


# ------------------------------------------------------------------------- n < 32: the generic_norm2 rule (H)
SMALL = {  # name -> (colour-2 values for m components, expected relation to the accurate norm)
    "sub_nonzero": lambda m, rng: rng.uniform(0.5, 1.5, m) * 1e-160,       # maxabs^2 subnormal: the lossy in-order sum
    "sq_zero": lambda m, rng: rng.uniform(0.5, 1.5, m) * 1e-170,           # maxabs^2 == 0: the scaled value
    "n_maxabs_inf": lambda m, rng: np.concatenate([[1.2e154], rng.uniform(0.5, 1.5, m - 1) * 1e150]),  # scaled
    "sq_overflow": lambda m, rng: rng.uniform(0.5, 1.5, m) * 1e300,         # the sum overflows: scaled
}


@pytest.mark.parametrize("n", [13, 31])
@pytest.mark.parametrize("small", list(SMALL))
@pytest.mark.parametrize("path,C,env", [("reg", 3, {}), ("lists", 10, {}), ("win", 10, {"NO_EPS_LISTS": 1})])
def test_fewer_than_32_components(pkg, oracle, dev, n, small, path, C, env):
    cv = cyc_colors(n, C)
    rng = np.random.default_rng(n)
    x = rng.uniform(0.5, 2.0, n)
    c2 = np.flatnonzero(cv == 2)
    x[c2] = SMALL[small](len(c2), rng) * np.where(rng.random(len(c2)) < 0.5, -1.0, 1.0)
    for fdtype, dir in MODES:
        eps = run(pkg, oracle, dev, x, fdtype, cv, dir=dir, absstep=0.0, env=env, colour2="finite")
        if small == "sub_nonzero":
            # the reference keeps the lossy sum; so must the device (an always-rescuing device would be more accurate)
            xm = np.where(cv == 2, x, 0.0)
            s = 0.0
            for v in xm:
                s += v * v
            assert s < 2.2250738585072014e-308
            np.testing.assert_allclose(abs(eps[1]), oracle.default_relstep(FD[fdtype]) * np.sqrt(np.sqrt(s)), rtol=1e-13)


# ---------------------------------------------------------------- default absstep with a tiny colour (I), per colour (J)
@pytest.mark.parametrize("C", [3, 20])
@pytest.mark.parametrize("fdtype,dir", MODES)
def test_default_absstep_tiny_colour(pkg, oracle, dev, C, fdtype, dir):
    N = 20_011
    cv = cyc_colors(N, C)
    for kind in ("sq_zero", "partly_sub", "below_T"):
        eps = run(pkg, oracle, dev, make_x(kind, cv), fdtype, cv, dir=dir, colour2="finite")
        relstep = oracle.default_relstep(FD[fdtype])              # the default absstep
        assert_same_bits(eps[1:2], np.array([relstep * (dir if fdtype == "forward" else 1.0)]), kind)


@pytest.mark.parametrize("case", ["sq_overflow", "norm_inf", "sq_zero", "trap", "mixed", "inf_in_big"])
@pytest.mark.parametrize("path,C,env", [("reg", 7, {}), ("lists", 20, {}), ("win", 20, {"NO_EPS_LISTS": 1})])
def test_rescue_is_per_colour(pkg, oracle, dev, case, path, C, env):
    N = 300_007 if case == "trap" else 20_011
    cv = colours(case, N, C)
    absstep, _ = CASES[case]
    x = make_x(case, cv)
    xin = x.copy()
    rng = np.random.default_rng(9)
    xin[cv == 2] = rng.uniform(0.5, 2.0, int((cv == 2).sum()))
    e = run(pkg, oracle, dev, x, "forward", cv, absstep=absstep, env=env)
    e_in = run(pkg, oracle, dev, xin, "forward", cv, absstep=absstep, env=env)
    assert_same_bits(np.delete(e, 1), np.delete(e_in, 1), "the in-range colours' step sizes")


# --------------------------------------------------------------- external step sizes and sharded groups (lists / reg)
@pytest.mark.parametrize("case", ["sq_overflow", "mixed", "inf_in_big"])
@pytest.mark.parametrize("C", [3, 20])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_external_step_sizes_column_blocks(pkg, oracle, dev, case, C, fdtype):
    from finitediff_jl_b200 import distributed as fdist
    N = 20_011
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, C)
    x_np = make_x(case, cv)
    x = torch.from_numpy(x_np).to(dev)
    J, _, _, _ = problem(pkg, oracle, dev, "csc", N)
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    pkg.finite_difference_jacobian_(J, lambda dx, xx: f_t(dx, xx), x, cache)
    eps_full = cache._last_plan.eps()
    eps = fdist.EpsPlan(N, cv, fdtype, dev).compute(x)
    assert_same_bits(eps.cpu().numpy()[:C], eps_full, "EpsPlan == the unsharded plan's step sizes")
    Jb, _, _, _ = problem(pkg, oracle, dev, "csc", N)
    bounds = fdist.column_blocks(colptr, 3)

    def factory(r0, r1, x0, x1):
        def f(dx, xs):
            # rows [r0, r1) of the scaled stencil from the slice x[x0:x1]
            full = torch.zeros(N, dtype=torch.float64, device=dev)
            full[x0:x1] = xs
            out = torch.empty(N, dtype=torch.float64, device=dev)
            f_t(out, full)
            dx.copy_(out[r0:r1])
        return f
    for r in range(3):
        blk = fdist.ColumnBlockJacobian(Jb, cv, fdtype, bounds[r], bounds[r + 1], dev, factory)
        blk.run(x, eps)
    torch.cuda.synchronize()
    assert_same_bits(Jb.nzval, J.nzval, "column blocks == the unsharded J")


@pytest.mark.parametrize("case", ["sq_overflow", "mixed"])
@pytest.mark.parametrize("C", [3, 20])
def test_group_two_members_one_device(pkg, oracle, dev, case, C):
    from finitediff_jl_b200 import distributed as fdist
    import ctypes
    L = pkg._lib
    N = 20_011
    cv = cyc_colors(N, C)
    x_np = make_x(case, cv)
    x = torch.from_numpy(x_np).to(dev)
    J1, _, _, _ = problem(pkg, oracle, dev, "csc", N)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J1)
    c1 = L.TridiagCtx(N, 0)
    pkg.finite_difference_jacobian_(J1, pkg.NativeFn(ctypes.cast(L.synth().fdbs_tridiag, ctypes.c_void_p).value, c1),
                                    x, cache)
    J2, _, _, _ = problem(pkg, oracle, dev, "csc", N)
    ctxs = [L.TridiagCtx(N, 0) for _ in range(2)]
    fs = [pkg.NativeFn(ctypes.cast(L.synth().fdbs_tridiag, ctypes.c_void_p).value, c) for c in ctxs]
    g = fdist.GroupJacobian(J2, cv, "forward", [0, 0])
    g.run(fs, x)
    g.synchronize()
    for p in g.plans:
        assert_same_bits(p.eps(), cache._last_plan.eps(), "every member's step sizes == the unsharded plan's")
    assert_same_bits(J1.nzval, J2.nzval, "sharded == unsharded")
    assert not torch.isnan(J1.nzval).any()
    g.close()


# --------------------------------------------------------------------- dense branch (per component) and the JVP
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_dense_branch_extremes(pkg, oracle, dev, fdtype):
    # component_eps has no sum: max(relstep*|x_i|, absstep) at |x| up to 1.7e308 and subnormal with absstep = 0
    N = 400
    rng = np.random.default_rng(31)
    x_np = rng.uniform(0.5, 2.0, N)
    x_np[:100] = rng.uniform(0.1, 1.7, 100) * 10.0 ** rng.integers(250, 308, 100) * np.where(rng.random(100) < 0.5, -1, 1)
    x_np[100] = 1.7e308
    x_np[101:200] = 10.0 ** rng.uniform(-323, -300, 99)
    x_np[200:203] = [5e-324, -0.0, 0.0]
    for absstep in (None, 0.0):
        kw = {} if absstep is None else {"absstep": absstep}
        x = torch.from_numpy(x_np).to(dev)
        J = pkg.zeros_colmajor(N, N, dev)
        cache = pkg.JacobianCache(x, torch.zeros(N, dtype=torch.float64, device=dev), fdtype)
        pkg.finite_difference_jacobian_(J, lambda dx, xx: f_t(dx, xx), x, cache, **kw)
        ref = np.zeros(N * N)
        r = oracle.jacobian(oracle.Problem.dense(N, N), ref, f_np, x_np.copy(), fdtype=FD[fdtype], **kw)
        assert np.isfinite(r["eps"]).all()
        assert_same_bits(cache._last_plan.eps(), r["eps"], f"per-component steps, absstep={absstep}")
        assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, f"J, absstep={absstep}")


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_jvp_dot_overflow_gives_inf(pkg, oracle, dev, fdtype):
    # jvp.jl:252: sqrt(abs(dot(x, v))); the reference's ddot overflows as a plain sum does, so eps is Inf on both sides
    N = 3000
    rng = np.random.default_rng(41)
    x_np = rng.uniform(1e300, 2e300, N)
    v_np = rng.uniform(1e10, 2e10, N)
    assert np.isinf(np.dot(x_np, v_np))
    x, v = torch.from_numpy(x_np).to(dev), torch.from_numpy(v_np).to(dev)
    jvp = torch.full((N,), float("nan"), dtype=torch.float64, device=dev)
    cache = pkg.JVPCache(x, fdtype)
    pkg.finite_difference_jvp_(jvp, lambda dx, xx: f_t(dx, xx), x, v, cache)
    torch.cuda.synchronize()
    own = oracle.jvp(f_np, x_np.copy(), v_np.copy(), N, fdtype=FD[fdtype])
    assert float(cache._last_plan.eps()[0]) == own["eps"] == np.inf


if __name__ == "__main__" and "--trace-paths" in sys.argv:
    _trace_paths()
