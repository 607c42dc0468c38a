"""Multi-GPU gradients: distributed.GroupGradient, the dense group with m = 1 (run with -m gpu; one GPU is enough).

Device ordinals may repeat, so [0, 0], [0, 0, 0] and [0, 0, 0, 0] run on one GPU exactly what as many GPUs run: the
contiguous column blocks, f(x) once at the root in forward mode, every member storing its entries into ONE df, the
event joins.  With two GPUs the same tests also run over [0, 1] and [1, 0, 1].  Every df is bit-compared
(tests/_util.assert_same_bits: signed zeros differ, NaN is one class) with the C restatement (scalar_oracle/) and with
finite_difference_gradient_ on one device, with no tolerance."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env
from scalar_oracle import fd_scalar_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    so.build()
    so.lib()
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


def device_sets():
    sets = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets += [[0, 1], [1, 0, 1]]
    return sets


def blocks(n, world):
    """member r owns the columns j with j // ceil(n / world) == r: a restatement of the partition"""
    p = -(-n // world)
    owner = [j // p for j in range(n)]
    return [(owner.index(r), n - owner[::-1].index(r)) if r in owner else (n, n) for r in range(world)]


# ------------------------------------------------------------------------------------------------ problems
class Scalar:
    """fdbs_quartic (or fdbs_guarded) with one context per member and its CPU twin."""

    def __init__(self, pkg, n, name="quartic", seed=17):
        rng = np.random.default_rng(seed + n)
        self.pkg, self.n, self.name = pkg, n, name
        self.a = 0.5 + rng.random(n)
        self.w = rng.random(n) * 2 - 1
        self._dev = {}
        self.twin = so.SynthScalar(n, self.a, self.w, name=f"synth_{name}")

    def fn(self, d):
        """a fresh NativeFn (own call counter) whose data lives on device d"""
        L = self.pkg._lib
        if d not in self._dev:
            dev = torch.device("cuda", d)
            self._dev[d] = (torch.from_numpy(self.a).to(dev), torch.from_numpy(self.w).to(dev))
        da, dw = self._dev[d]
        ctx = L.ScalarCtx(self.n, da.data_ptr(), dw.data_ptr(), 0)
        return self.pkg.NativeFn(C.cast(getattr(L.synth(), f"fdbs_{self.name}"), C.c_void_p).value, ctx, keepalive=(da, dw))

    def x(self, d=0):
        x = torch.empty(max(self.n, 1), dtype=torch.float64, device=torch.device("cuda", d))[: self.n]
        if self.n:
            self.pkg._lib.synth().fdbs_fill_x(x.data_ptr(), self.n, 0xFACE + self.n, None)
        return x

    def oracle(self, xh, mode, fx=None, **kw):
        return so.gradient(self.twin.native(f"synth_{self.name}"), xh, so.CENTRAL if mode == "central" else so.FORWARD,
                           fx=fx, **kw)


MODES = ["forward", "forward, fx number", "forward, fx tensor", "central"]


def fdtype_of(mode):
    return "central" if mode == "central" else "forward"


def fx_arg(mode, value, device):
    if mode == "forward, fx number":
        return value
    if mode == "forward, fx tensor":
        return torch.full((1,), value, dtype=torch.float64, device=device)
    return None


def single_df(pkg, fn, x, mode, fx=None, relstep=None, absstep=None, dir=1.0, **kw):
    n = x.numel()
    if fx is None:
        cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device=x.device), x, fdtype_of(mode), **kw)
    else:
        cache = pkg.GradientCache(fx, None, None, torch.zeros_like(x), fdtype_of(mode), **kw)
    df = torch.full((n,), NAN, dtype=torch.float64, device=x.device)
    pkg.finite_difference_gradient_(df, fn, x, cache, relstep=relstep, absstep=absstep, dir=dir)
    torch.cuda.synchronize()
    return df


def group_df(fdist, prob, devices, x, mode, fx=None, relstep=None, absstep=None, dir=1.0, **kw):
    df = torch.full((prob.n,), NAN, dtype=torch.float64, device=x.device)
    fs = [prob.fn(d) for d in devices]
    g = fdist.GroupGradient(prob.n, devices, fdtype_of(mode), **kw)
    g.run(fs, x, df, fx, relstep=relstep, absstep=absstep, dir=dir)
    g.synchronize()
    return g, fs, df


def check_members(g, fs, n, mode, what):
    """partition, per-member calls and launches: f(x) once (member 0) unless fx is given, then each member's columns"""
    world = len(g.plans)
    b = blocks(n, world)
    total = 0
    for r, (plan, f) in enumerate(zip(g.plans, fs)):
        lo, hi = plan.dense_range()
        assert (lo, hi) == b[r] == g.columns[r], (what, r)
        per = (hi - lo) * (2 if mode == "central" else 1)
        cnt = plan.counters()
        assert cnt["f_points"] == plan.info()["fcalls_per_jacobian"] - (mode != "central") == per, (what, r)
        assert f.ctx.calls == per + (1 if r == 0 and mode == "forward" else 0), (what, r)
        total += f.ctx.calls
        if hi == lo:
            assert cnt["kernel_launches"] == 0 and cnt["f_invocations"] == 0, (what, r)
    assert total == {"forward": n + 1, "central": 2 * n}.get(mode, n), what


# ------------------------------------------------------------------------------------------------ bit parity
NS = [1, 2, 3, 31, 32, 33] + list(range(1021, 1030)) + [20000]
_ORACLE = {}


def oracle_cached(prob, xh, mode, fx):
    key = (prob.name, prob.n, mode, xh.tobytes())
    if key not in _ORACLE:
        _ORACLE[key] = prob.oracle(xh, mode, fx)
    return _ORACLE[key]


@pytest.mark.parametrize("max_batch", [1, 7, 4096])
@pytest.mark.parametrize("n", NS)
def test_group_gradient_bit_parity(pkg, fdist, n, max_batch):
    prob = Scalar(pkg, n)
    x = prob.x()
    xh = x.cpu().numpy().copy()
    fxv = prob.twin(xh)
    for mode in MODES:
        ref = oracle_cached(prob, xh, mode, fxv if "fx" in mode else None)
        df1 = single_df(pkg, prob.fn(0), x, mode, fx_arg(mode, fxv, x.device), max_batch=max_batch)
        assert_same_bits(df1, ref["df"], f"single plan n={n} {mode}", allow_nan=False)
        for devices in device_sets():
            what = f"n={n} {mode} max_batch={max_batch} devices={devices}"
            root = torch.device("cuda", devices[0])
            xr = x.to(root)
            g, fs, df = group_df(fdist, prob, devices, xr, mode, fx_arg(mode, fxv, root), max_batch=max_batch)
            assert_same_bits(df, ref["df"], f"{what}: df vs restatement", allow_nan=False)
            assert_same_bits(df, df1, f"{what}: df vs single plan", allow_nan=False)
            assert_same_bits(xr, xh, f"{what}: x modified")
            check_members(g, fs, n, mode, what)
            g.close()


def test_group_gradient_one_member_and_empty(pkg, fdist):
    """group [0] is the single plan; n = 0 makes no member write (df may be an empty tensor without storage)"""
    n = 33
    prob = Scalar(pkg, n)
    x = prob.x()
    for mode in MODES:
        fxv = prob.twin(x.cpu().numpy())
        df1 = single_df(pkg, prob.fn(0), x, mode, fx_arg(mode, fxv, x.device))
        g, fs, df = group_df(fdist, prob, [0], x, mode, fx_arg(mode, fxv, x.device))
        assert_same_bits(df, df1, f"[0] {mode}", allow_nan=False)
        check_members(g, fs, n, mode, f"[0] {mode}")
    empty = Scalar(pkg, 0)
    for mode in MODES:
        for devices in [[0]] + device_sets():
            x0 = torch.empty(0, dtype=torch.float64, device=torch.device("cuda", devices[0]))
            g, fs, df = group_df(fdist, empty, devices, x0, mode, fx_arg(mode, 1.5, x0.device))
            assert df.numel() == 0
            check_members(g, fs, 0, mode, f"n=0 {mode} {devices}")


# ------------------------------------------------------------------------------------------------ steps, dir, reduced grid
STEPS = [(None, None), (1e-3, None), (None, 1e-6), (1e-12, 1e-160), (0.0, None), (None, 0.0), (0.0, 0.0), (-1e-3, None)]


@pytest.mark.parametrize("dir", [1.0, -1.0, 0.3])
@pytest.mark.parametrize("n", [33, 1025])
def test_group_gradient_steps_and_dir(pkg, fdist, n, dir):
    prob = Scalar(pkg, n)
    x = prob.x()
    xh = x.cpu().numpy().copy()
    fxv = prob.twin(xh)
    for relstep, absstep in STEPS:
        for mode in MODES:
            fx = fxv if "fx" in mode else None
            ref = prob.oracle(xh, mode, fx, relstep=relstep, absstep=absstep, dir=dir)
            df1 = single_df(pkg, prob.fn(0), x, mode, fx_arg(mode, fxv, x.device), relstep, absstep, dir, max_batch=64)
            assert_same_bits(df1, ref["df"], f"single n={n} {mode} steps={relstep, absstep} dir={dir}")
            for devices in device_sets():
                what = f"n={n} {mode} steps={relstep, absstep} dir={dir} devices={devices}"
                root = torch.device("cuda", devices[0])
                g, fs, df = group_df(fdist, prob, devices, x.to(root), mode, fx_arg(mode, fxv, root), relstep, absstep,
                                     dir, max_batch=64)
                assert_same_bits(df, ref["df"], f"{what}: df vs restatement")
                assert_same_bits(df, df1, f"{what}: df vs single plan")
                g.close()


@pytest.mark.parametrize("n", [1029, 20000])
def test_group_gradient_sm_count_1(pkg, fdist, n):
    """FDB_SM_COUNT=1: every kernel's grid wraps over many tiles per block"""
    prob = Scalar(pkg, n)
    x = prob.x()
    xh = x.cpu().numpy().copy()
    with fdb_env(SM_COUNT=1):
        for mode in ("forward", "central"):
            ref = oracle_cached(prob, xh, mode, None)
            for devices in device_sets():
                g, fs, df = group_df(fdist, prob, devices, x.to(torch.device("cuda", devices[0])), mode, max_batch=4096)
                assert_same_bits(df, ref["df"], f"n={n} {mode} SM_COUNT=1 devices={devices}", allow_nan=False)
                g.close()


# ------------------------------------------------------------------------------------------------ IEEE edges
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1e-160, 1.0, -2.5]


@pytest.mark.parametrize("n", [5, 33, 1025])
def test_group_gradient_ieee_edges(pkg, fdist, n):
    prob = Scalar(pkg, n, name="guarded")
    rng = np.random.default_rng(n)
    for k, (relstep, absstep) in enumerate(STEPS):
        xh = rng.standard_normal(n) * 10.0 ** rng.integers(-2, 3, n)
        for j, i in enumerate(sorted({0, 1, n // 2, n - 2, n - 1, 31 % n, 32 % n, 33 % n})):
            xh[i] = EDGES[(k + j) % len(EDGES)]
        x = torch.from_numpy(xh).cuda()
        fxv = prob.twin(xh)
        for mode in MODES:
            ref = prob.oracle(xh, mode, fxv if "fx" in mode else None, relstep=relstep, absstep=absstep)
            df1 = single_df(pkg, prob.fn(0), x, mode, fx_arg(mode, fxv, x.device), relstep, absstep, max_batch=7)
            assert_same_bits(df1, ref["df"], f"n={n} {mode} steps={relstep, absstep}: single plan")
            for devices in device_sets():
                what = f"n={n} {mode} steps={relstep, absstep} devices={devices}"
                root = torch.device("cuda", devices[0])
                g, fs, df = group_df(fdist, prob, devices, x.to(root), mode, fx_arg(mode, fxv, root), relstep, absstep,
                                     max_batch=7)
                assert_same_bits(df, df1, f"{what}: df vs single plan")
                assert_same_bits(df, ref["df"], f"{what}: df vs restatement")
                check_members(g, fs, n, mode, what)
                g.close()


# ------------------------------------------------------------------------------------------------ ownership
@pytest.mark.parametrize("n", [3, 33, 1027])
def test_group_gradient_members_write_their_own_columns(pkg, fdist, n):
    """Member r run alone with the group's slab pointer (df + col_begin) writes exactly [col_begin, col_end) of a
    NaN-filled df; the values are the single plan's.  Then, with member r's f scaled by 2^r (central mode: the quotient
    scales exactly), each entry of the group's df carries the factor of the one member that owns it."""
    L = pkg._lib
    prob = Scalar(pkg, n)
    x = prob.x()
    xh = x.cpu().numpy().copy()
    fin = torch.tensor([prob.twin(xh)], dtype=torch.float64, device=x.device)
    for mode in ("forward", "central"):
        df1 = single_df(pkg, prob.fn(0), x, mode, max_batch=7).cpu().numpy()
        for devices in device_sets():
            g = fdist.GroupGradient(n, devices, fdtype_of(mode), max_batch=7)
            for r, plan in enumerate(g.plans):
                lo, hi = plan.dense_range()
                f = prob.fn(devices[r])
                dev = torch.device("cuda", devices[r])
                xr, df = x.to(dev), torch.full((n,), NAN, dtype=torch.float64, device=dev)
                finr = fin.to(dev) if mode == "forward" else None
                with torch.cuda.device(dev):
                    L.check(L.lib().fdb_jacobian(plan.handle, f.address, f.ctx_ptr, xr.data_ptr(), df.data_ptr() + 8 * lo,
                                                 None, None if finr is None else finr.data_ptr(), L.STEP_DEFAULT,
                                                 L.STEP_DEFAULT, 1.0, None))
                torch.cuda.synchronize(dev)
                got = df.cpu().numpy()
                what = f"n={n} {mode} devices={devices} member {r}"
                assert_same_bits(got[lo:hi], df1[lo:hi], what, allow_nan=False)
                assert np.isnan(got[:lo]).all() and np.isnan(got[hi:]).all(), f"{what}: wrote outside its columns"
                assert f.ctx.calls == (hi - lo) * (2 if mode == "central" else 1), what
            g.close()
    for devices in device_sets():
        root = torch.device("cuda", devices[0])

        def scaled(k, d):
            a, w = (torch.from_numpy(v).to(torch.device("cuda", d)) for v in (prob.a, prob.w))

            def f(v):                                      # (batch, n) -> (batch,), times 2^k: exact in every quotient
                s = (w * v).sum(1)
                return (2.0 ** k) * ((a * v ** 4).sum(1) + s * s)
            f.batched = True
            return f

        g = fdist.GroupGradient(n, devices, "central", max_batch=7)
        out = []
        for scale in (True, False):                         # the same batches twice: only the factors differ
            df = torch.full((n,), NAN, dtype=torch.float64, device=root)
            g.run([scaled(r if scale else 0, d) for r, d in enumerate(devices)], x.to(root), df)
            g.synchronize()
            out.append(df.cpu().numpy())
        factor = np.zeros(n)
        for r, (lo, hi) in enumerate(blocks(n, len(devices))):
            factor[lo:hi] = 2.0 ** r
        assert_same_bits(out[0], out[1] * factor, f"n={n} devices={devices}: owner factors", allow_nan=False)
        g.close()


# ------------------------------------------------------------------------------------------------ points each member sees
@pytest.mark.parametrize("max_batch", [1, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 9])
def test_group_gradient_points_seen_by_members(pkg, fdist, n, max_batch):
    """each member's f sees its own columns' points in the reference's order (batched: a batch's + points, then, in
    central mode, its - points); the root's f first sees x itself in forward mode, and only there"""
    rng = np.random.default_rng(n)
    xh = rng.standard_normal(n)
    cube = lambda v: float(np.sum(v * v * v))
    for mode in ("forward", "central", "forward, fx number"):
        code = so.CENTRAL if mode == "central" else so.FORWARD
        fxv = cube(xh) if "fx" in mode else None
        ref = so.gradient(cube, xh, code, fx=fxv, log=True)
        pts = ref["points"]
        for devices in device_sets():
            seen = [[] for _ in devices]

            def make(k):
                def f(v):
                    seen[k].extend(v.cpu().numpy().copy())
                    return (v * v * v).sum(1)
                f.batched = True
                return f

            root = torch.device("cuda", devices[0])
            x = torch.from_numpy(xh).to(root)
            df = torch.full((n,), NAN, dtype=torch.float64, device=root)
            g = fdist.GroupGradient(n, devices, fdtype_of(mode), max_batch=max_batch)
            g.run([make(k) for k in range(len(devices))], x, df, fxv)
            g.synchronize()
            for r, (lo, hi) in enumerate(blocks(n, len(devices))):
                want = [pts[0]] if r == 0 and mode == "forward" else []
                shift = 1 if fxv is None and code == so.FORWARD else 0
                for c0 in range(lo, hi, max_batch):
                    cols = range(c0, min(hi, c0 + max_batch))
                    if code == so.CENTRAL:
                        want += [pts[2 * j] for j in cols] + [pts[2 * j + 1] for j in cols]
                    else:
                        want += [pts[shift + j] for j in cols]
                what = f"n={n} {mode} max_batch={max_batch} devices={devices} member {r}"
                assert len(seen[r]) == len(want), what
                for k, (p, q) in enumerate(zip(seen[r], want)):
                    assert_same_bits(p, q, f"{what} point {k}", allow_nan=False)
            assert sum(len(s) for s in seen) == ref["fcalls"]
            np.testing.assert_allclose(df.cpu().numpy(), 3 * xh * xh, rtol=1e-5, atol=1e-6)
            g.close()


# ------------------------------------------------------------------------------------------------ graph replay
def test_group_gradient_graph_replay_follows_x_and_fx(pkg, fdist):
    n = 1025
    prob = Scalar(pkg, n)
    for mode in MODES:
        for devices in device_sets():
            root = torch.device("cuda", devices[0])
            x = prob.x().to(root)
            df = torch.full((n,), NAN, dtype=torch.float64, device=root)
            fs = [prob.fn(d) for d in devices]
            fx_t = torch.full((1,), NAN, dtype=torch.float64, device=root)
            g = fdist.GroupGradient(n, devices, fdtype_of(mode), max_batch=64, use_graph=True)
            for k in range(3):
                x.mul_(1.0 + 0.125 * k)                 # written in place: the captured graphs read the same buffers
                xh = x.cpu().numpy().copy()
                fxv = prob.twin(xh)
                fx = None
                if mode == "forward, fx tensor":
                    fx_t.fill_(fxv)                      # written in place too
                    fx = fx_t
                elif mode == "forward, fx number":
                    fx = fxv
                df.fill_(NAN)
                g.run(fs, x, df, fx)
                g.synchronize()
                ref = prob.oracle(xh, mode, fxv if "fx" in mode else None)
                assert_same_bits(df, ref["df"], f"{mode} devices={devices} replay {k}", allow_nan=False)
            for plan in g.plans:
                assert plan.counters()["jacobians"] == 3
            g.close()


# ------------------------------------------------------------------------------------------------ errors
def test_group_gradient_errors(pkg, fdist):
    L = pkg._lib
    n = 8
    prob = Scalar(pkg, n)
    x = prob.x()
    df = torch.zeros(n, dtype=torch.float64, device="cuda")
    # complex step: the group builds, and fdb_group_jacobian refuses it before any f call
    g = fdist.GroupGradient(n, [0, 0], "complex")
    fs = [prob.fn(0), prob.fn(0)]
    with pytest.raises(L.FdbError) as e:
        g.run(fs, x, df)
    assert e.value.status == L.FDB_ERR_UNSUPPORTED
    assert fs[0].ctx.calls == fs[1].ctx.calls == 0
    g.close()
    g = fdist.GroupGradient(n, [0, 0], "forward")
    fs = [prob.fn(0), prob.fn(0)]
    bad = [
        ((fs[:1], x, df), ValueError),                                               # one f per member
        ((fs, x[:-1], df), ValueError),
        ((fs, x, df[:-1]), ValueError),
        ((fs, x.float(), df), TypeError),
        ((fs, x, df.float()), TypeError),
        ((fs, x.cpu(), df), TypeError),
        ((fs, x, df.cpu()), TypeError),
        ((fs, x, torch.zeros(2 * n, dtype=torch.float64, device="cuda")[::2]), ValueError),     # not contiguous
        ((fs, x, df, torch.zeros(2, dtype=torch.float64, device="cuda")), TypeError),
        ((fs, x, df, torch.zeros(1, dtype=torch.float32, device="cuda")), TypeError),
        ((fs, x, df, torch.zeros(1, dtype=torch.float64)), TypeError),
        ((fs, x, df, "1.0"), TypeError),
    ]
    if torch.cuda.device_count() >= 2:
        bad += [((fs, x.to("cuda:1"), df), ValueError), ((fs, x, df.to("cuda:1")), ValueError)]
    for args, exc in bad:
        with pytest.raises(exc):
            g.run(*args)
    assert fs[0].ctx.calls == fs[1].ctx.calls == 0

    # a failing native member, and a Python exception in any member (the root's f(x) included)
    fail = pkg.NativeFn(C.cast(L.synth().fdbs_fail, C.c_void_p).value)
    with pytest.raises(L.FdbError) as e:
        g.run([fail, fail], x, df)
    assert e.value.status == L.FDB_ERR_CALLBACK

    class Boom(Exception):
        pass

    def boom(v):
        raise Boom()

    ok = lambda v: (v * v).sum()
    for mode, fs_ in (("forward", [boom, ok]), ("forward", [ok, boom]), ("central", [ok, boom]), ("central", [boom, ok])):
        gg = fdist.GroupGradient(n, [0, 0], mode)
        torch.cuda.synchronize()
        with pytest.raises(Boom):
            gg.run(fs_, x, df)
        torch.cuda.synchronize()
        gg.close()
    with pytest.raises(ValueError):
        fdist.GroupGradient(-1, [0, 0])
    with pytest.raises(ValueError):
        fdist.GroupGradient(n, [0, 0], "hcentral")
    g.close()
