"""The block-banded plan (fdb_plan_create_block_banded / fdb_group_create_block_banded): BandedBlockBandedMatrix band data
written by a closed-form scatter, held bit for bit to the slot-addressed route it replaces (fdb_plan_create_coo on the
hook's entry list, run in the same process) and to the CPU oracle fed the device step sizes.

Every comparison prefills J with NaN: the new plan must write every one of the w*n slots, and the COO route (zero fill,
then scatter) defines every slot too, so the two buffers are compared whole, NaN counted as one class."""
import ctypes as C
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, fdb_env  # noqa: E402

FD = {"forward": 0, "central": 1, "complex": 2}


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


DEV = "cuda:0"


def _bbb(pkg, rb, l, u, lam, mu, dense_blocks=False):
    if dense_blocks:
        B = pkg.BlockBandedMatrix(rb, rb, (l, u), device=DEV)
    else:
        B = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device=DEV)
    B.data.fill_(float("nan"))
    return B


def _valid_coloring(B, rng):
    """A random distance-2 colouring of B's structure (greedy over a random column order)."""
    rows, cols, _ = B.findstructralnz()
    n = B.n
    by_col = [[] for _ in range(n)]
    for r, c in zip(rows.tolist(), cols.tolist()):
        by_col[c - 1].append(r - 1)
    row_cols = [[] for _ in range(B.m)]
    for c in range(n):
        for r in by_col[c]:
            row_cols[r].append(c)
    cv = np.zeros(n, np.int64)
    for c in rng.permutation(n):
        used = {int(cv[o]) for r in by_col[c] for o in row_cols[r] if cv[o] > 0}
        k = 1
        while k in used:
            k += 1
        cv[c] = k
    return cv


def _colorings(B, rng):
    """matrix_colors, 1:n, a random valid one, one with empty colours, one with columns the colour loop never reaches."""
    n = B.n
    mc = B.matrix_colors()
    rv = _valid_coloring(B, rng)
    gaps = 2 * rv + 1                                   # colours 2, 4, ... hold no column
    inval = rv.copy()
    inval[rng.random(n) < 0.3] = 0                      # colour 0 / negative: never perturbed, entries stay 0
    if n > 1:
        inval[rng.integers(0, n)] = -4
    return {"matrix_colors": mc, "identity": np.arange(1, n + 1, dtype=np.int64), "random": rv, "gaps": gaps,
            "invalid": inval}


class _Tri:
    """The native tridiagonal f! (any n), with its call counter."""

    def __init__(self, pkg, n, complex_=False):
        L = pkg._lib
        self.ctx = L.TridiagCtx(n, 0)
        sym = L.synth().fdbs_tridiag_c if complex_ else L.synth().fdbs_tridiag
        self.fn = pkg.NativeFn(C.cast(sym, C.c_void_p).value, self.ctx)


def _run(pkg, api, B, f, x, fdtype, cv, coo, **kw):
    """One Jacobian into B through the mirror: the block-banded plan, or (coo=True) the slot-addressed route the mirror
    took before it, on the entry list of findstructralnz."""
    run_kw = {k: kw.pop(k) for k in ("relstep", "absstep", "dir", "f_in") if k in kw}
    f_in = run_kw.pop("f_in", None)
    if coo:
        saved = api._block_banded_plan_args
        api._block_banded_plan_args = lambda J, sp: None
    try:
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B, **kw)
        pkg.finite_difference_jacobian_(B, f, x, cache, f_in, **run_kw)
    finally:
        if coo:
            api._block_banded_plan_args = saved
    torch.cuda.synchronize()
    return cache._last_plan


def _structure_cases():
    rng = np.random.default_rng(2024)
    cases = []
    for i in range(36):
        N = int(rng.integers(1, 13))
        rb = [int(b) for b in rng.integers(1, 10, N)]
        l, u = int(rng.integers(0, 4)), int(rng.integers(0, 4))
        lam, mu = int(rng.integers(0, 5)), int(rng.integers(0, 5))
        cases.append((i, rb, l, u, lam, mu, i % 9 == 8))
    # uniform blocks (no block lookup) and sub-bandwidths wider than a block
    cases.append((100, [4] * 7, 1, 1, 1, 1, False))
    cases.append((101, [3] * 5, 2, 0, 6, 7, False))
    cases.append((102, [1] * 9, 3, 2, 0, 0, False))
    return cases


STRUCTS = _structure_cases()


@pytest.mark.parametrize("case", STRUCTS, ids=[f"s{c[0]}" for c in STRUCTS])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_matches_coo_route_and_oracle(pkg, api, oracle, case, fdtype):
    _, rb, l, u, lam, mu, dense_blocks = case
    rng = np.random.default_rng(3 * case[0] + FD[fdtype])
    B = _bbb(pkg, rb, l, u, lam, mu, dense_blocks)
    n = B.n
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0x5EED + case[0], None)
    for name, cv in _colorings(B, rng).items():
        runs = [{}]
        if fdtype != "complex":
            runs += [{"relstep": 1e-5, "absstep": 1e-9}, {"absstep": 0.0}]
        if fdtype == "forward":
            runs += [{"dir": -1.0}, {"dir": 0.3}, {"f_in": "given"}]
        for kw in runs:
            got = {}
            for coo in (False, True):
                Bk = _bbb(pkg, rb, l, u, lam, mu, dense_blocks)
                f = _Tri(pkg, n, fdtype == "complex")
                kk = dict(kw)
                if kk.get("f_in") == "given":
                    # f(x) by the same native f (its 16-byte path wants even leading dimensions)
                    fx = torch.empty(n + 1, dtype=torch.float64, device=DEV)
                    fctx = pkg._lib.TridiagCtx(n, 0)
                    ld = (n + 1) & ~1
                    assert pkg._lib.synth().fdbs_tridiag(C.addressof(fctx), fx.data_ptr(), x.data_ptr(), 1, ld, ld, None) == 0
                    torch.cuda.synchronize()
                    kk["f_in"] = fx[:n]
                plan = _run(pkg, api, Bk, f.fn, x, fdtype, cv, coo, **kk)
                got[coo] = (Bk.data.cpu().numpy(), f.ctx.calls, plan)
            what = f"{case} {fdtype} {name} {kw}"
            info = got[False][2].info()
            assert info["jkind"] == pkg._lib.FDB_J_BLOCK_BAND, what
            assert got[True][2].info()["jkind"] == pkg._lib.FDB_J_SLOTS, what
            assert info["n_entries"] == len(B.findstructralnz()[0]), what
            assert_same_bits(got[False][0], got[True][0], what)
            assert not np.isnan(got[False][0]).any(), what
            assert got[False][1] == got[True][1], what
            if fdtype == "complex":
                continue
            rows, cols, slots = B.findstructralnz()
            refJ = np.full(B.w * n, np.nan)
            r = oracle.jacobian(oracle.Problem.coo_to_slots(n, n, rows, cols, slots, B.w * n), refJ,
                                oracle.native_fn("synth_tridiag"), oracle.fill_x(n, 0x5EED + case[0]),
                                fdtype=FD[fdtype], colorvec=cv, eps_override=got[False][2].eps(),
                                relstep=kw.get("relstep"), absstep=kw.get("absstep"), dir=kw.get("dir", 1.0),
                                f_in=None if kw.get("f_in") is None else kk["f_in"].cpu().numpy(),
                                ctx=oracle.SynthTridiagCtx(n, 1))
            assert_same_bits(got[False][0], refJ, what + " vs oracle")
            assert r["fcalls"] == got[False][1], what


def _traced_f(log):
    def f(fx, x):
        log.append(x.detach().cpu().numpy().copy())
        fx.copy_(x * x * x + 0.5 * torch.roll(x, 1))
    return f


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("max_batch", [1, 2, 5])
def test_same_points_and_order_as_coo_route(pkg, api, fdtype, max_batch):
    B = _bbb(pkg, [3, 5, 2, 4], 1, 1, 1, 2)
    n = B.n
    x = torch.linspace(-2.0, 3.0, n, dtype=torch.float64, device=DEV)
    cv = B.matrix_colors()
    out = {}
    for coo in (False, True):
        log = []
        Bk = _bbb(pkg, [3, 5, 2, 4], 1, 1, 1, 2)
        _run(pkg, api, Bk, _traced_f(log), x, fdtype, cv, coo, max_batch=max_batch)
        out[coo] = (Bk.data.cpu().numpy(), log)
    assert_same_bits(out[False][0], out[True][0])
    assert len(out[False][1]) == len(out[True][1])
    for a, b in zip(out[False][1], out[True][1]):
        assert_same_bits(a, b, "point passed to f")


TILE_CASES = [
    ([1] * 1023, 0, 0, 0, 0), ([1] * 1024, 0, 0, 0, 0), ([1] * 1025, 0, 0, 0, 0), ([2] * 1024, 0, 0, 0, 1),
    ([1] * 113, 1, 1, 1, 1), ([1] * 114, 1, 1, 1, 1), ([3] * 38, 1, 1, 1, 1), ([7, 5, 9] * 20, 1, 1, 1, 1),
]


@pytest.mark.parametrize("case", TILE_CASES, ids=[f"t{i}" for i in range(len(TILE_CASES))])
@pytest.mark.parametrize("passes", ["one", "batch1", "batch2", "few_slabs", "sm1"])
def test_tiles_and_colour_passes(pkg, api, case, passes):
    rb, l, u, lam, mu = case
    B = _bbb(pkg, rb, l, u, lam, mu)
    n = B.n
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 91, None)
    cv = B.matrix_colors()
    kw = {"one": {}, "batch1": {"max_batch": 1}, "batch2": {"max_batch": 2},
          "few_slabs": {"scratch_bytes": 8 * ((n + 1) & ~1) * 2}, "sm1": {}}[passes]
    res = {}
    for coo in (False, True):
        Bk = _bbb(pkg, rb, l, u, lam, mu)
        f = _Tri(pkg, n)
        if passes == "sm1":
            with fdb_env(FDB_SM_COUNT="1"):
                plan = _run(pkg, api, Bk, f.fn, x, "central", cv, coo, **kw)
        else:
            plan = _run(pkg, api, Bk, f.fn, x, "central", cv, coo, **kw)
        res[coo] = Bk.data.cpu().numpy()
        if passes == "few_slabs" and not coo and int(cv.max()) > 2:
            assert plan.info()["n_groups"] > 1
    assert_same_bits(res[False], res[True], f"{case} {passes}", allow_nan=False)


def test_graph_replay_after_x_changes_in_place(pkg, api):
    rb = [4, 6, 5, 4, 6]
    B = _bbb(pkg, rb, 1, 2, 2, 1)
    n = B.n
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    cv = B.matrix_colors()
    f = _Tri(pkg, n)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, use_graph=True)
    for seed in (5, 6, 7):
        pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, seed, None)   # x changes in place: the graph is replayed
        B.data.fill_(float("nan"))
        pkg.finite_difference_jacobian_(B, f.fn, x, cache)
        torch.cuda.synchronize()
        ref = _bbb(pkg, rb, 1, 2, 2, 1)
        _run(pkg, api, ref, _Tri(pkg, n).fn, x, "forward", cv, True)
        assert_same_bits(B.data.cpu().numpy(), ref.data.cpu().numpy(), f"seed {seed}", allow_nan=False)
    # the callback runs on the host once, while the call is captured; the replays run its launches only
    assert f.ctx.calls == 1 + int(cv.max())
    cnt = cache._last_plan.counters()
    assert cnt["jacobians"] == 3 and cnt["f_points"] == 3 * (1 + int(cv.max()))


def _lap5(pkg, g):
    n = g * g
    B = pkg.BandedBlockBandedMatrix([g] * g, [g] * g, (1, 1), (1, 1), device=DEV)
    B.data.fill_(float("nan"))
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0x1AB5, None)
    ctx = pkg._lib.Lap5Ctx(g, 0)
    f = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_lap5, C.c_void_p).value, ctx)
    return B, x, ctx, f


def test_lap5_g300_matches_coo_route(pkg, api):
    g = 300
    out = {}
    for coo in (False, True):
        B, x, ctx, f = _lap5(pkg, g)
        cv = B.matrix_colors()
        _run(pkg, api, B, f, x, "forward", cv, coo)
        out[coo] = (B.data.cpu().numpy(), ctx.calls)
    assert_same_bits(out[False][0], out[True][0], allow_nan=False)
    assert out[False][1] == out[True][1] == 10


def _stencil_coef(g, rows, cols):
    """d lap5(x)[row] / d x[col] of the synthetic 5-point stencil (clamped edges)."""
    i, j = rows % g, rows // g
    ip, jp = cols % g, cols // g
    coef = ((ip == i) & (jp == j)).astype(np.float64)
    coef += (ip == np.maximum(i - 1, 0)) & (jp == j)
    coef += (ip == np.minimum(i + 1, g - 1)) & (jp == j)
    coef += (ip == i) & (jp == np.maximum(j - 1, 0))
    coef += (ip == i) & (jp == np.minimum(j + 1, g - 1))
    return coef


@pytest.mark.parametrize("g", [1000, 3000])
def test_lap5_at_scale_sampled(pkg, g):
    n = g * g
    B, x, ctx, f = _lap5(pkg, g)
    cv = B.matrix_colors()
    t0 = time.perf_counter()
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, no_drift=1)
    plan = cache.plan_for(B, B, cache.colorvec, n)
    t_plan = time.perf_counter() - t0
    assert t_plan < 1.0, f"plan build took {t_plan:.3f} s"
    assert B._nz is None                                  # no host entry list was built
    pkg.finite_difference_jacobian_(B, f, x, cache)
    torch.cuda.synchronize()
    assert ctx.calls == 10
    data = B.data
    assert not torch.isnan(data).any().item()
    rng = np.random.default_rng(g)
    s = np.unique(rng.integers(0, 9 * n, 400_000))
    v = data[torch.from_numpy(s).to(DEV)].cpu().numpy()
    c = s // 9
    t = s % 9
    b, d = t // 3, t % 3
    J, j = c // g, c % g
    K, k = J + b - 1, j + d - 1
    inside = (K >= 0) & (K < g) & (k >= 0) & (k < g)
    # outside the structure (and the matrix): exactly +0.0
    assert np.all(v[~inside].view(np.uint64) == 0)
    rows = K[inside] * g + k[inside]
    coef = _stencil_coef(g, rows, c[inside])
    np.testing.assert_allclose(v[inside], coef, rtol=1e-6, atol=1e-6)
    # slots of the structure the stencil does not reach: f's row is unchanged, the quotient is exactly +0.0
    assert np.all(v[inside][coef == 0].view(np.uint64) == 0)


def device_sets():
    sets = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets += [[0, 1], [1, 0, 1]]
    return sets


@pytest.mark.parametrize("devices", device_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("partition", [0, 1])
def test_group_bit_identical_to_one_device(pkg, api, fdist, devices, fdtype, partition):
    root = torch.device("cuda", devices[0])
    cases = [([5, 3, 7, 4, 6, 2], 1, 2, 2, 1, "matrix_colors"), ([4] * 6, 1, 1, 1, 1, "matrix_colors"),
             ([3, 4, 2], 0, 1, 0, 0, "few"), ([6, 2, 5, 4], 2, 1, 3, 2, "invalid")]
    for rb, l, u, lam, mu, kind in cases:
        B1 = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device=root)
        n = B1.n
        if kind == "few":        # one colour: fewer colours than members
            cv = np.ones(n, np.int64)
        elif kind == "invalid":
            cv = _valid_coloring(B1, np.random.default_rng(3))
            cv[::3] = 0
        else:
            cv = B1.matrix_colors()
        x = torch.empty(n, dtype=torch.float64, device=root)
        pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 17, None)
        # one device, the new plan, and the COO route
        B1.data.fill_(float("nan"))
        one = _Tri(pkg, n)
        with torch.cuda.device(root):
            cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B1)
            pkg.finite_difference_jacobian_(B1, one.fn, x, cache)
        torch.cuda.synchronize(root)
        # the group
        BG = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device=root)
        BG.data.fill_(float("nan"))
        ctxs = [_Tri(pkg, n) for _ in devices]
        gj = fdist.GroupJacobian(BG, cv, fdtype, devices, partition=partition)
        gj.run([c.fn for c in ctxs], x)
        gj.synchronize()
        what = f"{devices} {rb} {kind} partition={partition}"
        assert_same_bits(BG.data.cpu().numpy(), B1.data.cpu().numpy(), what, allow_nan=False)
        # per-member calls: forward members evaluate f(x) and their own colours
        owner = gj.plans[0].color_owner()
        C_ = int(max(cv.max(), 0))
        for i, c in enumerate(ctxs):
            own = int(np.sum(owner == i))
            expect = 1 + own if fdtype == "forward" else 2 * own
            assert c.ctx.calls == expect, (what, i)
            assert gj.plans[i].info()["jkind"] == pkg._lib.FDB_J_BLOCK_BAND
        assert sum(int(np.sum(owner == i)) for i in range(len(devices))) == C_
        gj.close()


def test_group_complex_refused(pkg, fdist):
    B = pkg.BandedBlockBandedMatrix([3, 3], [3, 3], (1, 1), (1, 1), device=DEV)
    cv = B.matrix_colors()
    x = torch.ones(B.n, dtype=torch.float64, device=DEV)
    gj = fdist.GroupJacobian(B, cv, "complex", [0, 0])
    f = _Tri(pkg, B.n, True)
    with pytest.raises(pkg._lib.FdbError) as e:
        gj.run([f.fn, f.fn], x)
    assert e.value.status == pkg._lib.FDB_ERR_UNSUPPORTED
    gj.close()


def test_refusals(pkg):
    L = pkg._lib
    lib = L.lib()
    o = L.PlanOpts()
    h = C.c_void_p()

    def create(blocks, l=1, u=1, lam=1, mu=1, ldata=None, nblocks=None):
        b = np.asarray(blocks, np.int64)
        n = int(b.sum()) if len(b) else 0
        w = (l + u + 1) * (lam + mu + 1)
        return lib.fdb_plan_create_block_banded(C.byref(h), len(b) if nblocks is None else nblocks,
                                                b.ctypes.data if len(b) else None, l, u, lam, mu,
                                                w * n if ldata is None else ldata, None, C.byref(o))

    assert create([3, -1, 4]) == L.FDB_ERR_INVALID
    assert create([3, 3], l=-1) == L.FDB_ERR_INVALID
    assert create([3, 3], mu=-2) == L.FDB_ERR_INVALID
    assert create([3, 3], ldata=9 * 6 - 1) == L.FDB_ERR_INVALID
    assert lib.fdb_plan_create_block_banded(C.byref(h), 2, None, 1, 1, 1, 1, 54, None, C.byref(o)) == L.FDB_ERR_INVALID
    assert lib.fdb_plan_create_block_banded(None, 1, np.array([2], np.int64).ctypes.data, 0, 0, 0, 0, 2, None,
                                            C.byref(o)) == L.FDB_ERR_INVALID
    assert create([3, 3]) == L.FDB_OK
    p = pkg.Plan(h.value)
    assert lib.fdb_plan_set_peers(p.handle, 0, None) == L.FDB_ERR_UNSUPPORTED
    assert p.info()["j_len"] == 54 and p.info()["jkind"] == L.FDB_J_BLOCK_BAND
    # no block at all: an empty matrix
    assert create([]) == L.FDB_OK
    pkg.Plan(h.value)


def test_rectangular_and_dense_targets_keep_the_coo_route(pkg, api, oracle):
    # rectangular block lists: the mirror's slot-addressed route, unchanged
    B = pkg.BandedBlockBandedMatrix([3, 4, 2], [2, 5, 2], (1, 1), (1, 0), device=DEV)
    assert api._block_banded_plan_args(B, B) is None
    n = B.n
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 3, None)
    f = _Tri(pkg, n)
    cv = np.arange(1, n + 1, dtype=np.int64)
    B.data.fill_(float("nan"))
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B)
    pkg.finite_difference_jacobian_(B, f.fn, x, cache)
    torch.cuda.synchronize()
    assert cache._last_plan.info()["jkind"] == pkg._lib.FDB_J_SLOTS
    rows, cols, slots = B.findstructralnz()
    ref = np.full(B.w * n, np.nan)
    oracle.jacobian(oracle.Problem.coo_to_slots(B.m, n, rows, cols, slots, B.w * n), ref, oracle.native_fn("synth_tridiag"),
                    oracle.fill_x(n, 3), colorvec=cv, eps_override=cache._last_plan.eps(), ctx=oracle.SynthTridiagCtx(n, 1))
    assert_same_bits(B.data.cpu().numpy(), ref)
    # a dense J with a block-banded sparsity: the COO route into the dense matrix
    S = pkg.BandedBlockBandedMatrix([3, 4], [3, 4], (1, 1), (1, 1), device=DEV)
    assert api._block_banded_plan_args(pkg.zeros_colmajor(7, 7, DEV), S) is None
