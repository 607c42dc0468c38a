"""Multi-GPU Hessians: rank/world Hessian plans and fdb_group_hessian (run with -m gpu; one GPU is enough).

Device ordinals may repeat, so [0, 0], [0, 0, 0] and [0, 0, 0, 0] run on one GPU exactly what as many GPUs run: the
point-balanced split of the i-blocks, f(x) once per non-empty member, every member storing its entries into ONE H,
the event joins.  With two GPUs the same tests also run over [0, 1] and [1, 0, 1].  Every H is bit-compared
(tests/_util.assert_same_bits: signed zeros differ, NaN is one class) with the C restatement (scalar_oracle/) and
with the single-plan GPU H, with no tolerance."""
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


# ------------------------------------------------------------------------------------------------ the partition, restated
def block_start(i, n):
    return 1 + 2 * i + 4 * (i * (n - 1) - i * (i - 1) // 2)


def partition(n, world):
    """[i_0 = 0, ..., i_world = n]: i_r is the i in [i_{r-1}, n] whose S(i) - 1 is nearest to r * 2n^2 / world (exact
    rational distance), ties to the smaller i — a linear scan, independent of the library's binary search."""
    T = 2 * n * n
    b = [0]
    for r in range(1, world):
        best, best_d = None, None
        for i in range(b[-1], n + 1):
            d = abs(world * (block_start(i, n) - 1) - r * T)
            if best_d is None or d < best_d:
                best, best_d = i, d
        b.append(best)
    b.append(n)
    return b


def member_points(n, b, r):
    """f evaluations of rank r: f(x) and its points, none for an empty rank > 0"""
    own = block_start(b[r + 1], n) - block_start(b[r], n)
    return 0 if (r > 0 and b[r] == b[r + 1]) else 1 + own


def owned_mask(n, lo, hi):
    m = np.zeros((n, n), dtype=bool)
    for i in range(lo, hi):
        m[i:, i] = True          # column i, rows [i, n)
        m[i, i + 1:] = True      # row i, columns (i, n)
    return m


# ------------------------------------------------------------------------------------------------ problems
class Scalar:
    """fdbs_quartic (or fdbs_guarded) with one context per device and its CPU twin."""

    def __init__(self, pkg, n, name="quartic", seed=7):
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
            self.pkg._lib.synth().fdbs_fill_x(x.data_ptr(), self.n, 0xC0FFEE + self.n, None)
        return x


def strided_H(n, ld, d=0):
    """H viewed in a NaN-filled buffer with leading dimension ld: column j of H = buf[j][:n]"""
    buf = torch.full((max(n, 1), max(ld, 1)), NAN, dtype=torch.float64, device=torch.device("cuda", d))
    H = buf[:n, :n].t() if n else torch.empty((0, 0), dtype=torch.float64, device=torch.device("cuda", d))
    return H, buf


def single_H(pkg, fn, x, relstep=None, absstep=None, **kw):
    n = x.numel()
    H, _ = strided_H(n, n, x.device.index)
    pkg.finite_difference_hessian_(H, fn, x, pkg.HessianCache(x, **kw), relstep=relstep, absstep=absstep)
    torch.cuda.synchronize()
    return H


def group_H(fdist, prob, devices, x, ld, relstep=None, absstep=None, reps=1, **kw):
    n = prob.n
    H, buf = strided_H(n, ld, devices[0])
    fx = torch.full((1,), NAN, dtype=torch.float64, device=x.device)
    fs = [prob.fn(d) for d in devices]
    g = fdist.GroupHessian(n, devices, ldH=max(ld, 1), **kw)
    for _ in range(reps):
        g.run(fs, x, H, fx, relstep=relstep, absstep=absstep)
    g.synchronize()
    return g, fs, H, buf, fx


_ORACLE = {}


def oracle_quartic(prob, xh):
    key = (prob.name, prob.n, xh.tobytes())
    if key not in _ORACLE:
        _ORACLE[key] = so.hessian(prob.twin.native(f"synth_{prob.name}"), xh)
    return _ORACLE[key]


# ------------------------------------------------------------------------------------------------ bit parity, calls, partition
@pytest.mark.parametrize("max_batch", [1, 7, 4096])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 31, 32, 33, 65, 257])
def test_group_hessian_bit_parity(pkg, fdist, n, max_batch):
    prob = Scalar(pkg, n)
    x = prob.x()
    xh = x.cpu().numpy().copy()
    ref = oracle_quartic(prob, xh)
    H1 = single_H(pkg, prob.fn(0), x, max_batch=max_batch)
    assert_same_bits(H1, ref["H"][:n, :n], f"single plan n={n}", allow_nan=False)
    for devices in device_sets():
        what = f"n={n} max_batch={max_batch} devices={devices}"
        root = torch.device("cuda", devices[0])
        xr = x.to(root)
        g, fs, H, buf, fx = group_H(fdist, prob, devices, xr, n + 3, max_batch=max_batch)
        assert_same_bits(H, ref["H"][:n, :n], f"{what}: H vs restatement", allow_nan=False)
        assert_same_bits(H, H1, f"{what}: H vs single plan", allow_nan=False)
        assert torch.isnan(buf[:, n:]).all(), f"{what}: padding rows written"
        assert_same_bits(fx, np.array([ref["fx"]]), f"{what}: f(x)", allow_nan=False)
        assert_same_bits(xr, xh, f"{what}: x modified")
        b = partition(n, len(devices))
        entries = 0
        for r, (plan, f) in enumerate(zip(g.plans, fs)):
            assert plan.dense_range() == (b[r], b[r + 1]), what
            info, cnt = plan.info(), plan.counters()
            pts = member_points(n, b, r)
            assert f.ctx.calls == cnt["f_points"] == info["fcalls_per_jacobian"] == pts, (what, r)
            assert info["n_entries"] == int(owned_mask(n, b[r], b[r + 1]).sum()), (what, r)
            entries += info["n_entries"]
            if pts == 0:
                assert cnt["kernel_launches"] == 0 and cnt["f_invocations"] == 0, (what, r)
        assert entries == n * n, what
        g.close()


def test_group_hessian_n1000_matches_single_plan(pkg, fdist):
    n = 1000
    prob = Scalar(pkg, n)
    x = prob.x()
    H1 = single_H(pkg, prob.fn(0), x, max_batch=4096)
    for devices in device_sets():
        _, fs, H, _, fx = group_H(fdist, prob, devices, x.to(torch.device("cuda", devices[0])), n, max_batch=4096)
        assert_same_bits(H, H1, f"n=1000 devices={devices}", allow_nan=False)
        assert sum(f.ctx.calls for f in fs) == 2 * n * n + len(devices)      # every member is non-empty here


@pytest.mark.parametrize("world", [1, 2, 3, 4, 7, 64])
def test_rank_plan_partition(pkg, world):
    """fdb_plan_dense_range of every rank tiles [0, n), equals the restated rule, and each rank's point count is within
    one i-block of T/world; plan_info's counts sum to the whole Hessian's plus one f(x) per non-empty rank > 0."""
    L = pkg._lib
    for n in (0, 1, 2, 3, 5, 8, 31, 100, 1000, 2049):
        b = partition(n, world)
        got = []
        fcalls = entries = 0
        for r in range(world):
            h = C.c_void_p()
            o = L.PlanOpts(fdtype=L.FDB_HCENTRAL, rank=r, world=world, max_batch=64, scratch_bytes=1 << 20)
            L.check(L.lib().fdb_hessian_plan_create(C.byref(h), n, n, C.byref(o)))
            p = pkg.Plan(h.value)
            got.append(p.dense_range())
            info = p.info()
            fcalls += info["fcalls_per_jacobian"]
            entries += info["n_entries"]
            assert info["fcalls_per_jacobian"] == member_points(n, b, r)
            p.destroy()
        assert got == [(b[r], b[r + 1]) for r in range(world)], (n, world, got, b)
        assert b == sorted(b) and b[0] == 0 and b[-1] == n
        extra = sum(1 for r in range(1, world) if b[r] < b[r + 1])
        assert fcalls == 2 * n * n + 1 + extra and entries == n * n, (n, world)
        for r in range(world):
            pts = block_start(b[r + 1], n) - block_start(b[r], n)
            assert abs(world * pts - 2 * n * n) <= world * (2 + 4 * max(n - 1, 0)), (n, world, r)


@pytest.mark.parametrize("n,case", [(65, "chunks"), (257, "chunks"), (65, "sm1"), (257, "sm1")])
def test_group_hessian_chunks_and_reduced_grid(pkg, fdist, n, case):
    """small scratch_bytes: every non-empty member runs several value chunks; FDB_SM_COUNT=1: the assembly and patch
    grids wrap over many tiles per block"""
    prob = Scalar(pkg, n)
    x = prob.x()
    ref = oracle_quartic(prob, x.cpu().numpy().copy())
    ldx = max(2, (n + 1) & ~1)
    # 8 batch rows take half the budget; the value buffer holds 8 ldx - 1 values besides f(x)
    kw = {"max_batch": 8, "scratch_bytes": 16 * 8 * ldx} if case == "chunks" else {"max_batch": 7}
    with fdb_env(SM_COUNT=1 if case == "sm1" else None):
        for devices in device_sets():
            g, _, H, _, _ = group_H(fdist, prob, devices, x.to(torch.device("cuda", devices[0])), n, **kw)
            assert_same_bits(H, ref["H"], f"n={n} {case} devices={devices}", allow_nan=False)
            if case == "chunks":
                b = partition(n, len(devices))
                for r, plan in enumerate(g.plans):
                    own = block_start(b[r + 1], n) - block_start(b[r], n)
                    assert own > 8 * ldx - 1 and plan.info()["n_groups"] > 1, (devices, r, own)
            g.close()


# ------------------------------------------------------------------------------------------------ points each member sees
@pytest.mark.parametrize("max_batch", [1, 5])
@pytest.mark.parametrize("n", [1, 2, 4, 5])
def test_group_hessian_points_seen_by_members(pkg, fdist, n, max_batch):
    rng = np.random.default_rng(n)
    xh = rng.standard_normal(n)
    ref = so.hessian(lambda v: float(np.sum(v * v * v)), xh, log=True)
    for devices in device_sets():
        seen = [[] for _ in devices]

        def make(k):
            def f(v):
                seen[k].append(v.cpu().numpy().copy())
                return (v * v * v).sum()
            return f

        root = torch.device("cuda", devices[0])
        x = torch.from_numpy(xh).to(root)
        H = pkg.zeros_colmajor(n, n, root)
        g = fdist.GroupHessian(n, devices, max_batch=max_batch)
        g.run([make(k) for k in range(len(devices))], x, H)
        g.synchronize()
        b = partition(n, len(devices))
        for r in range(len(devices)):
            want = [] if member_points(n, b, r) == 0 else \
                [ref["points"][0]] + ref["points"][block_start(b[r], n):block_start(b[r + 1], n)]
            assert len(seen[r]) == len(want), (devices, r)
            for k, (p, q) in enumerate(zip(seen[r], want)):
                assert_same_bits(p, q, f"devices={devices} member {r} point {k}", allow_nan=False)
        np.testing.assert_allclose(H.cpu().numpy(), np.diag(6 * xh), atol=1e-5)
        g.close()


# ------------------------------------------------------------------------------------------------ graph replay
def test_group_hessian_graph_replay_follows_x(pkg, fdist):
    n = 33
    prob = Scalar(pkg, n)
    for devices in device_sets():
        root = torch.device("cuda", devices[0])
        x = prob.x().to(root)
        H, _ = strided_H(n, n, devices[0])
        fx = torch.full((1,), NAN, dtype=torch.float64, device=root)
        fs = [prob.fn(d) for d in devices]
        g = fdist.GroupHessian(n, devices, max_batch=64, use_graph=True)
        for k in range(3):
            x.mul_(1.0 + 0.125 * k)                 # written in place: the captured graphs read the same buffer
            H.fill_(NAN)
            g.run(fs, x, H, fx)
            g.synchronize()
            ref = so.hessian(prob.twin.native("synth_quartic"), x.cpu().numpy().copy())
            assert_same_bits(H, ref["H"], f"devices={devices} replay {k}", allow_nan=False)
            assert_same_bits(fx, np.array([ref["fx"]]), f"devices={devices} replay {k}: f(x)", allow_nan=False)
        for r, plan in enumerate(g.plans):
            assert plan.counters()["jacobians"] == 3
        g.close()


# ------------------------------------------------------------------------------------------------ IEEE edges
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1e-160, 1.0, -2.5]
STEPS = [(None, None), (None, 0.0), (0.0, None), (1e-12, 1e-160), (None, 1e-320), (-1e-3, None)]


@pytest.mark.parametrize("n", [5, 33, 65])
def test_group_hessian_ieee_edges(pkg, fdist, n):
    prob = Scalar(pkg, n, name="guarded")
    rng = np.random.default_rng(n)
    for k, (relstep, absstep) in enumerate(STEPS):
        xh = rng.standard_normal(n) * 10.0 ** rng.integers(-2, 3, n)
        for j, i in enumerate(sorted({0, 1, n // 2, n - 2, n - 1, 31 % n, 32 % n})):
            xh[i] = EDGES[(k + j) % len(EDGES)]
        x = torch.from_numpy(xh).cuda()
        H1 = single_H(pkg, prob.fn(0), x, relstep, absstep, max_batch=7)
        ref = so.hessian(prob.twin.native("synth_guarded"), xh, relstep=relstep, absstep=absstep)
        assert_same_bits(H1, ref["H"], f"n={n} steps={relstep, absstep}: single plan")
        for devices in device_sets():
            what = f"n={n} steps={relstep, absstep} devices={devices}"
            root = torch.device("cuda", devices[0])
            _, _, H, _, fx = group_H(fdist, prob, devices, x.to(root), n, relstep, absstep, max_batch=7)
            assert_same_bits(H, H1, f"{what}: H vs single plan")
            assert_same_bits(fx, np.array([ref["fx"]]), f"{what}: f(x)")


# ------------------------------------------------------------------------------------------------ rank plans without a group
def test_rank_plans_share_one_H_on_two_streams(pkg):
    n = 97
    prob = Scalar(pkg, n)
    x = prob.x()
    H1 = single_H(pkg, prob.fn(0), x, max_batch=64)
    H, _ = strided_H(n, n)
    caches = [pkg.HessianCache(x, max_batch=64, rank=r, world=2) for r in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        pkg.finite_difference_hessian_(H, prob.fn(0), x, caches[r], stream=streams[r].cuda_stream)
    torch.cuda.synchronize()
    assert_same_bits(H, H1, "two rank plans, one H", allow_nan=False)
    b = partition(n, 2)
    for r in range(2):
        assert caches[r]._last_plan.dense_range() == (b[r], b[r + 1])
        # one rank alone writes exactly its own entries
        H, _ = strided_H(n, n)
        fx = torch.full((1,), NAN, dtype=torch.float64, device="cuda")
        pkg.finite_difference_hessian_(H, prob.fn(0), x, caches[r], fx=fx)
        torch.cuda.synchronize()
        m = owned_mask(n, b[r], b[r + 1])
        got, want = H.cpu().numpy(), H1.cpu().numpy()
        assert_same_bits(got[m], want[m], f"rank {r}: owned entries", allow_nan=False)
        assert np.isnan(got[~m]).all(), f"rank {r} wrote entries it does not own"
        assert_same_bits(fx, np.array([oracle_quartic(prob, x.cpu().numpy().copy())["fx"]]), f"rank {r}: f(x)")


# ------------------------------------------------------------------------------------------------ errors
def test_group_hessian_errors(pkg, fdist):
    L = pkg._lib
    lib = L.lib()
    n = 8
    prob = Scalar(pkg, n)
    x = prob.x()
    H = pkg.zeros_colmajor(n, n)
    devs = (C.c_int * 2)(0, 0)
    # fdtype other than hcentral
    for bad in (L.FDB_FORWARD, L.FDB_CENTRAL, L.FDB_COMPLEX):
        h = C.c_void_p()
        assert lib.fdb_group_create_hessian(C.byref(h), 2, devs, n, n, C.byref(L.PlanOpts(fdtype=bad))) == L.FDB_ERR_UNSUPPORTED
    with pytest.raises(L.FdbError) as e:
        fdist.GroupHessian(n, [0, 0], fdtype="central")
    assert e.value.status == L.FDB_ERR_UNSUPPORTED
    # cross-kind calls, before any launch
    g = fdist.GroupHessian(n, [0, 0])
    fs = [prob.fn(0), prob.fn(0)]
    ctxs = (C.c_void_p * 2)(C.cast(fs[0].ctx_ptr, C.c_void_p).value, C.cast(fs[1].ctx_ptr, C.c_void_p).value)
    assert lib.fdb_group_jacobian(g._h, fs[0].address, ctxs, x.data_ptr(), H.data_ptr(), None, None, L.STEP_DEFAULT,
                                  L.STEP_DEFAULT, 1.0, None) == L.FDB_ERR_INVALID
    assert fs[0].ctx.calls == fs[1].ctx.calls == 0
    J = pkg.zeros_colmajor(n, n)
    gj = C.c_void_p()
    L.check(lib.fdb_group_create_dense(C.byref(gj), 2, devs, n, n, n, C.byref(L.PlanOpts(fdtype=L.FDB_CENTRAL))))
    assert lib.fdb_group_hessian(gj, fs[0].address, ctxs, x.data_ptr(), J.data_ptr(), None, L.STEP_DEFAULT, L.STEP_DEFAULT,
                                 None) == L.FDB_ERR_INVALID
    lib.fdb_group_destroy(gj)
    assert fs[0].ctx.calls == fs[1].ctx.calls == 0
    # a failing native member
    fail = pkg.NativeFn(C.cast(L.synth().fdbs_fail, C.c_void_p).value)
    with pytest.raises(L.FdbError) as e:
        g.run([fail, fail], x, H)
    assert e.value.status == L.FDB_ERR_CALLBACK

    # a Python exception in one member's f
    class Boom(Exception):
        pass

    def boom(v):
        raise Boom()

    torch.cuda.synchronize()
    with pytest.raises(Boom):
        g.run([lambda v: (v * v).sum(), boom], x, H)
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        g.run([prob.fn(0)], x, H)                              # one f per member
    g.close()
