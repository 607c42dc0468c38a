"""Multi-GPU out-of-place Jacobians: out-of-place rank plans and fdb_group_jacobian_oop (run with -m gpu; one GPU is
enough).

Device ordinals may repeat, so [0, 0], [0, 0, 0] and [0, 0, 0, 0] run on one GPU exactly what as many GPUs run: the
colour partition (dense branch: column blocks), every member writing its own slots of ONE result, the root's zero fill
and compaction, the event joins.  With two GPUs the same tests also run over [0, 1] and [1, 0, 1].  Every result is
bit-compared (tests/_util.assert_same_bits) with the C restatement oop_oracle/ (fed the device step sizes for coloured
plans, as tests/test_gpu_oop.py does) and with the one-device result, with no tolerance.  The ownership rules are
checked one rank plan at a time on results prefilled with -0.0, where a stray `+ 0.0` or zero store shows."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env, tridiag_csc
from oop_oracle import fd_oop_oracle as OO
from test_gpu_oop import NpF, TorchF, _sparse_proto, _to_host_result, _x, assert_same_result, f_masked, f_nl

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
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
def restated_owner(C, world, counts, mode):
    """0: colour k on rank k mod world; 1: LPT, heaviest colour first (ties: smaller colour) onto the least-loaded rank
    (ties: smaller rank), a colour of c entries weighing c + 1"""
    owner = np.zeros(C, np.int32)
    if world == 1:
        return owner
    if mode == 0:
        return (np.arange(C) % world).astype(np.int32)
    load = [0] * world
    for k in sorted(range(C), key=lambda k: (-counts[k], k)):
        r = min(range(world), key=lambda r: (load[r], r))
        owner[k] = r
        load[r] += counts[k] + 1
    return owner


def restated_blocks(C, world):
    per = -(-C // world)
    return [(min(C, per * r), min(C, per * r + per)) for r in range(world)]


# ------------------------------------------------------------------------------------------------ problems
KINDS = ["raw", "dense_proto", "sparse_proto", "csc_dense", "csc_sparse"]


def _problem(pkg, kind, n, cv=None, m=None):
    """(torch kwargs, oracle kwargs, colorvec, C) of a result kind: the tridiagonal pattern (cyclic colours 1:3 unless cv)
    with a sparsity, else the dense branch over C = maximum(cv) quotient columns (1:n unless cv)"""
    m = n if m is None else m
    if kind in ("raw", "dense_proto", "sparse_proto"):
        tk, lk = ({"colorvec": cv}, {"colorvec": cv}) if cv is not None else ({}, {})
        C_ = n if cv is None else int(max(cv))
        if kind == "dense_proto":
            tk["jac_prototype"] = torch.zeros((C_ + 2, m), dtype=torch.float64, device="cuda").t()
            lk["jac_prototype"] = ("dense", m, C_ + 2)
        elif kind == "sparse_proto":
            tk["jac_prototype"] = _sparse_proto(pkg, m, C_ + 2)
            lk["jac_prototype"] = ("sparse", m, C_ + 2)
        return tk, lk, cv, C_
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64) if cv is None else cv
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    tk = {"sparsity": S, "colorvec": cv}
    lk = {"sparsity": (n, n, cp, rv), "colorvec": cv}
    if kind == "csc_sparse":
        tk["jac_prototype"] = S
        lk["jac_prototype"] = ("sparse", n, n)
    return tk, lk, cv, int(max(cv.max(), 0))


def _entry_counts(n, cv, C):
    cp, _ = tridiag_csc(n)
    per_col = np.diff(cp)
    return [int(per_col[cv == k + 1].sum()) for k in range(C)]


def _colour_owner(g, kind, n, cv, C, partition):
    """owner member of every colour (dense branch: column), restated, and checked against the plans"""
    world = len(g.devices)
    if kind.startswith("csc"):
        want = restated_owner(C, world, _entry_counts(n, cv, C), partition)
        for p in g.plans:
            assert np.array_equal(p.color_owner()[:C], want), "fdb_plan_color_owner != the restated partition"
        return want
    blocks = restated_blocks(C, world)
    for p, b in zip(g.plans, blocks):
        assert p.dense_range() == b, "fdb_plan_dense_range != the restated column blocks"
    owner = np.zeros(C, np.int32)
    for r, (b0, b1) in enumerate(blocks):
        owner[b0:b1] = r
    return owner


def _group(fdist, devs, kind, fd, tk, partition=0, **kw):
    return fdist.GroupJacobianOOP(devs, fd, colorvec=tk.get("colorvec"), sparsity=tk.get("sparsity"),
                                  jac_prototype=tk.get("jac_prototype"), partition=partition, **kw)


def _single(pkg, kind, fd, fn, xd, tk, dir, relstep, absstep, f_in):
    cache = pkg.JacobianCache(xd, fd)
    fin = fn(xd) if f_in else None
    res = pkg.finite_difference_jacobian(TorchF(fn, False), xd, cache, fin, relstep=relstep, absstep=absstep, dir=dir,
                                         **tk)
    eps = list(cache._last_plan.eps()) if kind.startswith("csc") else None
    return res, eps


def _expected_points(nf_points, fd, owner, r, root_fx):
    """the oracle's point sequence restricted to member r's colours; root_fx: the root's own f(x) comes first"""
    pts = list(nf_points)
    out = []
    if root_fx:
        x0, pts = pts[0], pts[1:]
        if r == 0:
            out.append(x0)
    per = 2 if fd == "central" else 1
    for k in range(len(owner)):
        if owner[k] == r:
            out += pts[per * k: per * k + per]
    return out


def _check_member_points(fs, nf, fd, owner, root_fx, what):
    for r, f in enumerate(fs):
        want = _expected_points(nf.points, fd, owner, r, root_fx)
        assert len(f.points) == len(want), f"{what}: member {r} saw {len(f.points)} points, expected {len(want)}"
        for i, (a, b) in enumerate(zip(f.points, want)):
            assert_same_bits(a, b, f"{what}: member {r} point {i}")


def _parity(pkg, fdist, devs, kind, fd, *, n=13, dir=1.0, steps=(None, None), f_in=False, partition=0, cv=None,
            fn=f_nl, x=None, record=True):
    tk, lk, cv, C = _problem(pkg, kind, n, cv)
    x = _x(n, seed=n + len(devs)) if x is None else x
    xd = torch.from_numpy(x).cuda(devs[0])
    x_before = xd.clone()
    relstep, absstep = steps
    with torch.cuda.device(devs[0]):
        single, eps = _single(pkg, kind, fd, fn, xd, tk, dir, relstep, absstep, f_in)
        g = _group(fdist, devs, kind, fd, tk, partition)
        fs = [TorchF(fn, record) for _ in devs]
        fin = fn(xd) if f_in else None
        res = g.run(fs, xd, fin, relstep=relstep, absstep=absstep, dir=dir)
        torch.cuda.synchronize()
    what = f"{devs} {kind} {fd} dir={dir} steps={steps} f_in={f_in} partition={partition}"
    assert_same_bits(xd, x_before, f"{what}: the caller's x")
    rel = pkg.default_relstep(fd) if relstep is None else relstep
    nf = NpF(fn)
    want = OO.jacobian_oop(nf, x, fd, fn(x, np) if f_in else None, relstep=rel, absstep=absstep, dir=dir,
                           eps_override=eps, **lk)
    assert_same_result(res, want, f"{what}: against the restatement")
    assert_same_result(res, _to_host_result(single), f"{what}: against one device")
    if record:
        owner = _colour_owner(g, kind, n, cv, C, partition)
        # through the mirror, forward mode: f(x) is evaluated once, by the root's f, and passed on as f_in
        if fd == "forward" and not f_in:
            assert len(fs[0].points) >= 1 and len(nf.points) == 1 + C
        _check_member_points(fs, nf, fd, owner, fd == "forward" and not f_in, what)
        total = sum(len(f.points) for f in fs)
        assert total == (2 * C if fd == "central" else C + (0 if f_in else 1)), f"{what}: {total} calls in all"
    g.close()
    return res


# ------------------------------------------------------------------------------------------------ parity
CASES = [("forward", 1.0, (None, None), False), ("forward", -1.0, (1e-3, 0.0), False), ("forward", 0.3, (0.0, 1e-4), True),
         ("central", 1.0, (None, None), False), ("central", -1.0, (1e-2, None), False), ("central", 0.3, (None, 1e-4), True)]


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fd,dir,steps,f_in", CASES)
def test_group_parity(pkg, fdist, devs, kind, fd, dir, steps, f_in):
    _parity(pkg, fdist, devs, kind, fd, dir=dir, steps=steps, f_in=f_in)


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("kind", ["csc_dense", "csc_sparse"])
@pytest.mark.parametrize("fd", ["forward", "central"])
def test_group_lpt_partition(pkg, fdist, devs, kind, fd):
    """LPT over colours of uneven weight: a sparse result takes any colouring (1, 2, 2, 3, 3, 3, ... columns per colour);
    a dense one needs a valid colouring, the cyclic 1:4, whose colours hold 8, 7, 7 and 7 columns at n = 29"""
    n = 29
    if kind == "csc_sparse":
        cv = np.array([1, 2, 2, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 5] * 2, np.int64)[:n]
    else:
        cv = (np.arange(n) % 4 + 1).astype(np.int64)
    _parity(pkg, fdist, devs, kind, fd, n=n, partition=1, cv=cv, dir=-1.0)


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("fd", ["forward", "central"])
def test_group_colourless_columns(pkg, fdist, devs, fd):
    """columns without a valid colour (colour 0) in a sparse result: their candidates are rank 0's zeros, and dropped"""
    n = 31
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    cv[::5] = 0
    for kind in ("csc_sparse",):
        _parity(pkg, fdist, devs, kind, fd, n=n, cv=cv)
    # no valid colour at all: nobody evaluates a colour, the root writes every candidate's zero
    res = _parity(pkg, fdist, devs, "csc_sparse", fd, n=n, cv=np.zeros(n, np.int64))
    assert res.nnz == 0


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("kind", ["raw", "dense_proto", "sparse_proto"])
def test_group_fewer_columns_than_members(pkg, fdist, devs, kind):
    """dense branch with C = 2 < world on the wider device sets: the members past the blocks are empty"""
    n = 9
    cv = np.array([1, 2, 1, 2, 1, 2, 1, 2, 1], np.int64)
    for fd in ("forward", "central"):
        _parity(pkg, fdist, devs, kind, fd, n=n, cv=cv)


@pytest.mark.parametrize("n", [341, 342, 343])
@pytest.mark.parametrize("sm", [None, 1])
def test_group_tile_edges(pkg, fdist, n, sm):
    """3n - 2 = 1021, 1024, 1027 candidates of the CSC sparse result; m x C = 1023 .. 1029 on the dense branch"""
    with fdb_env(SM_COUNT=sm):
        _parity(pkg, fdist, [0, 0, 0], "csc_sparse", "forward", n=n, dir=-1.0, record=False)
        _parity(pkg, fdist, [0, 0], "csc_dense", "central", n=n, record=False)
        cv = (np.arange(n) % 3 + 1).astype(np.int64)
        _parity(pkg, fdist, [0, 0, 0], "sparse_proto", "forward", n=n, cv=cv, record=False)


def test_group_masked_zeros_and_nan(pkg, fdist):
    """exactly-zero quotients (dropped by the sparse kinds, +0.0 in the dense ones) and NaN (kept)"""
    n = 40
    mask = (np.arange(n) % 5 != 0).astype(np.float64)
    maskd = torch.from_numpy(mask).cuda()
    fn = lambda x, lib=torch: f_masked(x, mask if lib is np else maskd.to(x.device), lib)
    x = _x(n, seed=5)
    x[17] = np.nan
    for kind in KINDS:
        for dir in (1.0, -1.0):
            _parity(pkg, fdist, [0, 0, 0], kind, "forward", n=n, dir=dir, fn=fn, x=x)


# ------------------------------------------------------------------------------------------------ through the ABI
def _abi_group(pkg, devs, kind, n, cv, fd, proto_cols=None, **kw):
    L = pkg._lib
    o = pkg.api._opts(pkg.api._fdtype_code(fd), devs[0], **kw)
    d = (C.c_int * len(devs))(*devs)
    h = C.c_void_p()
    code = {"raw": L.FDB_OOP_RAW, "dense_proto": L.FDB_OOP_DENSE, "sparse_proto": L.FDB_OOP_SPARSE,
            "csc_dense": L.FDB_OOP_DENSE, "csc_sparse": L.FDB_OOP_SPARSE}[kind]
    if kind.startswith("csc"):
        cp, rv = tridiag_csc(n)
        L.check(L.lib().fdb_group_create_oop_csc(C.byref(h), len(devs), d, n, n, cp.ctypes.data, rv.ctypes.data,
                                                 cv.ctypes.data, code, n, C.byref(o)))
    else:
        L.check(L.lib().fdb_group_create_oop_dense(C.byref(h), len(devs), d, n, n, None if cv is None else cv.ctypes.data,
                                                   proto_cols or 0, code, n, C.byref(o)))
    return h


def _member_plans(pkg, h, k):
    out = []
    for i in range(k):
        p = C.c_void_p()
        pkg._lib.check(pkg._lib.lib().fdb_group_plan(h, i, C.byref(p)))
        out.append(pkg.Plan(p.value, owned=False))
    return out


def _trampolines(pkg, fs, n, devs):
    """one fdb_fn for every member (the ABI takes one entry point and a context per member)"""
    per = [pkg.api._PyFn(f, n, n, torch.device("cuda", d), False, oop=True) for f, d in zip(fs, devs)]

    def tramp(ctx, p_fx, p_x, batch, ldfx, ldx, stream, _per=per):
        return _per[int(ctx or 1) - 1]._tramp(None, p_fx, p_x, batch, ldfx, ldx, stream)

    keep = pkg._lib.FDB_FN(tramp)
    ctxs = (C.c_void_p * len(per))(*[i + 1 for i in range(len(per))])
    return pkg._lib.fn_address(keep), ctxs, (keep, per)


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("kind", ["csc_dense", "raw"])
@pytest.mark.parametrize("with_fin", [False, True])
def test_group_member_calls_and_launches(pkg, devs, kind, with_fin):
    """forward mode through the ABI: without f_in every non-empty member evaluates f(x) first, then its colours
    ascending; with f_in no member evaluates f(x) (members on another device read the replica); an empty member calls
    nothing and launches nothing"""
    L = pkg._lib
    n = 13
    cv = (np.arange(n) % 3 + 1).astype(np.int64) if kind.startswith("csc") else np.array([1, 2] * 6 + [1], np.int64)
    h = _abi_group(pkg, devs, kind, n, cv, "forward")
    try:
        plans = _member_plans(pkg, h, len(devs))
        x = _x(n, seed=2)
        xd = torch.from_numpy(x).cuda(devs[0])
        fs = [TorchF(f_nl) for _ in devs]
        addr, ctxs, keep = _trampolines(pkg, fs, n, devs)
        C_ = 3 if kind.startswith("csc") else 2
        ncols = n if kind.startswith("csc") else C_
        J = torch.full((ncols, n), NAN, dtype=torch.float64, device=xd.device).t()
        out = L.OopOut()
        out.J = J.data_ptr()
        # an f_in that is not f(x): members that evaluated f(x) instead of reading it would give other quotients
        fin = (f_nl(xd) + 0.25) if with_fin else None
        with torch.cuda.device(devs[0]):
            L.check(L.lib().fdb_group_jacobian_oop(h, addr, ctxs, xd.data_ptr(), C.byref(out), None,
                                                   None if fin is None else fin.data_ptr(), L.STEP_DEFAULT,
                                                   L.STEP_DEFAULT, 1.0, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        lk = {"colorvec": cv}
        if kind.startswith("csc"):
            cp, rv = tridiag_csc(n)
            lk["sparsity"] = (n, n, cp, rv)
        eps = list(plans[0].eps()) if kind.startswith("csc") else None
        nf = NpF(f_nl)
        want = OO.jacobian_oop(nf, x, "forward", None if fin is None else fin.cpu().numpy(), eps_override=eps, **lk)
        assert_same_bits(J.cpu().numpy(), want[1], f"{devs} {kind} f_in={with_fin}")
        if kind.startswith("csc"):
            owner = restated_owner(C_, len(devs), _entry_counts(n, cv, C_), 0)
        else:
            owner = np.zeros(C_, np.int32)
            for r, (b0, b1) in enumerate(restated_blocks(C_, len(devs))):
                owner[b0:b1] = r
        colour_pts = nf.points if with_fin else nf.points[1:]
        for r, (f, p) in enumerate(zip(fs, plans)):
            own = [k for k in range(C_) if owner[k] == r]
            cnt = p.counters()
            if r > 0 and not own:
                assert len(f.points) == 0 and cnt["f_points"] == 0 and cnt["kernel_launches"] == 0, f"member {r} is empty"
                assert p.info()["fcalls_per_jacobian"] == 0
                continue
            want_pts = ([] if with_fin else [x]) + [colour_pts[k] for k in own]
            assert len(f.points) == len(want_pts), f"member {r}: {len(f.points)} calls, expected {len(want_pts)}"
            for i, (a, b) in enumerate(zip(f.points, want_pts)):
                assert_same_bits(a, b, f"member {r} point {i}")
            assert p.info()["fcalls_per_jacobian"] == len(want_pts) + (1 if with_fin else 0)
            assert p.info()["n_local_colors"] == len(own)
    finally:
        L.lib().fdb_group_destroy(h)


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("fd", ["forward", "central"])
def test_group_root_zero_fills_a_dense_csc_result(pkg, devs, fd):
    """a NaN-prefilled J: the non-structural elements are +0.0 only because the root zero-fills J before the members"""
    L = pkg._lib
    n = 50
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    h = _abi_group(pkg, devs, "csc_dense", n, cv, fd)
    try:
        plans = _member_plans(pkg, h, len(devs))
        x = _x(n, seed=4)
        xd = torch.from_numpy(x).cuda(devs[0])
        addr, ctxs, keep = _trampolines(pkg, [TorchF(f_nl, False) for _ in devs], n, devs)
        J = torch.full((n, n), NAN, dtype=torch.float64, device=xd.device)
        out = L.OopOut()
        out.J = J.data_ptr()
        with torch.cuda.device(devs[0]):
            L.check(L.lib().fdb_group_jacobian_oop(h, addr, ctxs, xd.data_ptr(), C.byref(out), None, None, L.STEP_DEFAULT,
                                                   L.STEP_DEFAULT, -1.0, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        cp, rv = tridiag_csc(n)
        want = OO.jacobian_oop(NpF(f_nl), x, fd, dir=-1.0, colorvec=cv, sparsity=(n, n, cp, rv), eps_override=list(plans[0].eps()))
        assert_same_bits(J.t().cpu().numpy(), want[1], f"{devs} {fd}")
    finally:
        L.lib().fdb_group_destroy(h)


@pytest.mark.parametrize("devs", device_sets())
def test_group_sparse_outputs_and_capacity(pkg, devs):
    """NaN / -1 prefilled sparse outputs are fully defined where the result lives; a too small out->cap is refused before
    any call"""
    L = pkg._lib
    n = 60
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    h = _abi_group(pkg, devs, "csc_sparse", n, cv, "forward")
    try:
        plans = _member_plans(pkg, h, len(devs))
        assert plans[0].info()["n_entries"] == 3 * n - 2
        x = _x(n, seed=6)
        xd = torch.from_numpy(x).cuda(devs[0])
        fs = [TorchF(f_nl) for _ in devs]
        addr, ctxs, keep = _trampolines(pkg, fs, n, devs)
        E = 3 * n - 2
        cpo = torch.full((n + 1,), -1, dtype=torch.int64, device=xd.device)
        rvo = torch.full((E,), -1, dtype=torch.int64, device=xd.device)
        nzo = torch.full((E,), NAN, dtype=torch.float64, device=xd.device)
        nnz = torch.full((1,), -1, dtype=torch.int64, device=xd.device)
        out = L.OopOut()
        out.colptr, out.rowval, out.nzval, out.cap, out.nnz = cpo.data_ptr(), rvo.data_ptr(), nzo.data_ptr(), E - 1, nnz.data_ptr()
        stream = C.c_void_p(torch.cuda.current_stream(xd.device).cuda_stream)
        with torch.cuda.device(devs[0]):
            st = L.lib().fdb_group_jacobian_oop(h, addr, ctxs, xd.data_ptr(), C.byref(out), None, None, L.STEP_DEFAULT,
                                                L.STEP_DEFAULT, 1.0, stream)
            assert st == L.FDB_ERR_INVALID and b"capacity" in L.lib().fdb_last_error()
            assert all(len(f.points) == 0 for f in fs)
            out.cap = E
            L.check(L.lib().fdb_group_jacobian_oop(h, addr, ctxs, xd.data_ptr(), C.byref(out), None, None, L.STEP_DEFAULT,
                                                   L.STEP_DEFAULT, 1.0, stream))
        torch.cuda.synchronize()
        cp, rv = tridiag_csc(n)
        want = OO.jacobian_oop(NpF(f_nl), x, "forward", colorvec=cv, sparsity=(n, n, cp, rv),
                               jac_prototype=("sparse", n, n), eps_override=list(plans[0].eps()))
        k = int(nnz.item())
        assert np.array_equal(cpo.cpu().numpy(), want[3])
        assert np.array_equal(rvo[:k].cpu().numpy(), want[4])
        assert_same_bits(nzo[:k].cpu().numpy(), want[5], "nzval")
    finally:
        L.lib().fdb_group_destroy(h)


# ------------------------------------------------------------------------------------------------ ownership, one rank at a time
def _rank_plan(pkg, kind, n, cv, rank, world, fd="forward", proto_cols=None):
    """rank plans share the result (shared_j: they never zero-fill it); the one-device plan (world = 1) owns its own"""
    L = pkg._lib
    o = pkg.api._opts(pkg.api._fdtype_code(fd), 0, rank=rank, world=world, shared_j=world > 1)
    h = C.c_void_p()
    code = {"raw": L.FDB_OOP_RAW, "dense_proto": L.FDB_OOP_DENSE, "csc_dense": L.FDB_OOP_DENSE,
            "csc_sparse": L.FDB_OOP_SPARSE, "sparse_proto": L.FDB_OOP_SPARSE}[kind]
    if kind.startswith("csc"):
        cp, rv = tridiag_csc(n)
        L.check(L.lib().fdb_oop_plan_create_csc(C.byref(h), n, n, cp.ctypes.data, rv.ctypes.data, cv.ctypes.data, code, n,
                                                C.byref(o)))
    else:
        L.check(L.lib().fdb_oop_plan_create_dense(C.byref(h), n, n, None if cv is None else cv.ctypes.data,
                                                  proto_cols or 0, code, n, C.byref(o)))
    return pkg.Plan(h.value)


def _run_rank(pkg, plan, xd, J, f=None, stream=None):
    L = pkg._lib
    tf = f or TorchF(f_nl, False)
    n = xd.numel()
    addr, ctx, keep = pkg.api._as_fn(tf, n, n, xd.device, 1, oop=True)
    out = L.OopOut()
    out.J = J.data_ptr()
    s = stream if stream is not None else torch.cuda.current_stream()
    L.check(L.lib().fdb_jacobian_oop(plan.handle, addr, ctx, xd.data_ptr(), C.byref(out), None, None, L.STEP_DEFAULT,
                                     L.STEP_DEFAULT, 1.0, C.c_void_p(s.cuda_stream)))
    return keep


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("kind", ["csc_dense", "dense_proto", "raw"])
def test_rank_writes_exactly_its_own_slots(pkg, world, kind):
    """J prefilled with -0.0: a rank changes its own slots to the one-device values and leaves every other -0.0 alone
    (a `+ 0.0` over another rank's slot would turn it into +0.0).  The prototype's columns [C, ncols) are rank 0's."""
    n = 23
    cv = (np.arange(n) % 3 + 1).astype(np.int64) if kind == "csc_dense" else (np.arange(n) % 5 + 1).astype(np.int64)
    C_ = 3 if kind == "csc_dense" else 5
    ncols = n if kind == "csc_dense" else (C_ + 3 if kind == "dense_proto" else C_)
    xd = torch.from_numpy(_x(n, seed=9)).cuda()
    one = _rank_plan(pkg, kind, n, cv, 0, 1, proto_cols=ncols)
    J1 = torch.full((ncols, n), -0.0, dtype=torch.float64, device="cuda").t()
    _run_rank(pkg, one, xd, J1)
    torch.cuda.synchronize()
    ref = J1.cpu().numpy()
    cp, rv = tridiag_csc(n)
    col = np.repeat(np.arange(n), np.diff(cp))
    union = np.zeros((n, ncols), bool)
    for r in range(world):
        p = _rank_plan(pkg, kind, n, cv, r, world, proto_cols=ncols)
        J = torch.full((ncols, n), -0.0, dtype=torch.float64, device="cuda").t()
        _run_rank(pkg, p, xd, J)
        torch.cuda.synchronize()
        got = J.cpu().numpy()
        own = np.zeros((n, ncols), bool)
        if kind == "csc_dense":
            owner = restated_owner(C_, world, _entry_counts(n, cv, C_), 0)
            assert np.array_equal(p.color_owner()[:C_], owner)
            mine = owner[cv[col] - 1] == r
            own[rv[mine] - 1, col[mine]] = True
        else:
            b0, b1 = restated_blocks(C_, world)[r]
            assert p.dense_range() == (b0, b1)
            own[:, b0:b1] = True
            if r == 0:
                own[:, C_:] = True
        assert_same_bits(got[own], ref[own], f"{kind} rank {r}/{world}: its own slots")
        assert (np.signbit(got[~own]) & (got[~own] == 0)).all(), f"{kind} rank {r}/{world} wrote a slot it does not own"
        union |= own
    if kind == "csc_dense":
        struct = np.zeros((n, ncols), bool)
        struct[rv - 1, col] = True
        assert np.array_equal(union, struct)
    else:
        assert union.all()


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("kind", ["csc_sparse", "sparse_proto"])
def test_sparse_member_candidates_land_on_its_own_entries(pkg, fdist, devs, kind):
    """one member's f returns NaN: exactly the entries of that member's colours (dense branch: its column block) are NaN
    in the result, every other entry is the one-device value"""
    n = 17
    cv = (np.arange(n) % 3 + 1).astype(np.int64) if kind == "csc_sparse" else (np.arange(n) % 7 + 1).astype(np.int64)
    tk, lk, cv, C_ = _problem(pkg, kind, n, cv)
    xd = torch.from_numpy(_x(n, seed=12)).cuda(devs[0])
    with torch.cuda.device(devs[0]):
        single, _ = _single(pkg, kind, "central", f_nl, xd, tk, 1.0, None, None, False)
    sh = _to_host_result(single)
    for r in range(len(devs)):
        g = _group(fdist, devs, kind, "central", tk)
        fs = [TorchF((lambda v: f_nl(v) * NAN) if i == r else f_nl, False) for i in range(len(devs))]
        with torch.cuda.device(devs[0]):
            res = g.run(fs, xd)
        owner = _colour_owner(g, kind, n, cv, C_, 0)
        h = _to_host_result(res)
        # every candidate of member r is NaN (kept); the others are the one-device entries
        if kind == "csc_sparse":
            cp, rv = tridiag_csc(n)
            col = np.repeat(np.arange(n), np.diff(cp))
            mine = owner[cv[col] - 1] == r
            rows_cols_r = set(zip(rv[mine] - 1, col[mine]))
        else:
            rows_cols_r = {(i, c) for c in range(C_) if owner[c] == r for i in range(n)}
        gcol = np.repeat(np.arange(h[2]), np.diff(h[3]))
        grc = list(zip(h[4] - 1, gcol))
        nan_rc = {rc for rc, v in zip(grc, h[5]) if np.isnan(v)}
        assert nan_rc == rows_cols_r, f"{devs} {kind}: member {r}'s candidates"
        scol = np.repeat(np.arange(sh[2]), np.diff(sh[3]))
        sval = {rc: v for rc, v in zip(zip(sh[4] - 1, scol), sh[5])}
        for rc, v in zip(grc, h[5]):
            if rc not in rows_cols_r:
                assert_same_bits(np.array([v]), np.array([sval[rc]]), f"{devs} {kind}: entry {rc}")
        g.close()


def test_two_dense_rank_plans_on_two_streams_share_one_j(pkg):
    """standalone dense-kind rank plans: the owner zero-fills, the ranks run concurrently on two streams into one J"""
    for kind in ("csc_dense", "dense_proto"):
        n = 301
        cv = (np.arange(n) % 3 + 1).astype(np.int64)
        ncols = n if kind == "csc_dense" else 6
        xd = torch.from_numpy(_x(n, seed=21)).cuda()
        one = _rank_plan(pkg, kind, n, cv, 0, 1, proto_cols=ncols)
        J1 = torch.full((ncols, n), NAN, dtype=torch.float64, device="cuda").t()
        _run_rank(pkg, one, xd, J1)
        plans = [_rank_plan(pkg, kind, n, cv, r, 2, proto_cols=ncols) for r in range(2)]
        J = torch.zeros((ncols, n), dtype=torch.float64, device="cuda").t()       # the owner's zero fill
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        keep = [_run_rank(pkg, p, xd, J, stream=s) for p, s in zip(plans, streams)]
        torch.cuda.synchronize()
        assert_same_bits(J.cpu().numpy(), J1.cpu().numpy(), f"{kind}: two ranks on two streams")
        del keep


def test_group_graph_replay_after_x_changes(pkg, fdist):
    """use_graph: every member captures its call once and replays it while x changes in place (central mode and a
    sparse result: x, the candidate buffer and every scalar stay the same, so the graphs are reused)"""
    from oracle import fd_oracle as orc
    L = pkg._lib
    n = 4000
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), torch.zeros(len(rv), dtype=torch.float64,
                                                                                          device="cuda"))
    for devs in device_sets():
        xd = torch.from_numpy(_x(n, seed=1)).cuda(devs[0])
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, L.TridiagCtx(n, 0)) for _ in devs]
        g = fdist.GroupJacobianOOP(devs, "central", colorvec=cv, sparsity=S, jac_prototype=S, use_graph=True)
        with torch.cuda.device(devs[0]):
            for seed in (1, 2, 3):
                xd.copy_(torch.from_numpy(_x(n, seed=seed)))
                res = g.run(fs, xd, dir=-1.0)
                cache = pkg.JacobianCache(xd, "central")
                want = pkg.finite_difference_jacobian(fs[0], xd, cache, sparsity=S, colorvec=cv, jac_prototype=S, dir=-1.0)
                assert_same_result(res, _to_host_result(want), f"{devs} replay {seed}")
                twin = (C.cast(orc.native_fn("synth_tridiag"), C.c_void_p).value, orc.SynthTridiagCtx(n, 1))
                want = OO.jacobian_oop(twin, xd.cpu().numpy(), "central", sparsity=(n, n, cp, rv), colorvec=cv,
                                       jac_prototype=("sparse", n, n), dir=-1.0, eps_override=list(cache._last_plan.eps()))
                assert_same_result(res, want, f"{devs} replay {seed}: against the restatement")
        assert all(p.counters()["jacobians"] == 3 for p in g.plans if p.info()["n_local_colors"] > 0)
        g.close()


@pytest.mark.parametrize("devs", device_sets())
def test_group_c2_size_sparse_result(pkg, fdist, devs):
    """N = 10^7 tridiagonal, 3 colours, the native stencil fdbs_tridiag on every member: the group's sparse result is the
    one-device result and the C restatement's, bit for bit"""
    from oracle import fd_oracle as orc
    L = pkg._lib
    n = 10_000_000
    x = orc.fill_x(n, 0x5EED + 7)
    x[np.arange(5, n, 97)] = 2.0 ** 90
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    xd = torch.from_numpy(x).cuda(devs[0])
    fs = [pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, L.TridiagCtx(n, 0)) for _ in devs]
    with torch.cuda.device(devs[0]):
        for fd, dir in (("forward", 1.0), ("central", -1.0)):
            cache = pkg.JacobianCache(xd, fd)
            single = pkg.finite_difference_jacobian(fs[0], xd, cache, sparsity=S, colorvec=cv, jac_prototype=S, dir=dir)
            g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=S, jac_prototype=S)
            res = g.run(fs, xd, dir=dir)
            assert_same_result(res, _to_host_result(single), f"{devs} C2 {fd}: against one device")
            if fd == "forward":
                twin = (C.cast(orc.native_fn("synth_tridiag"), C.c_void_p).value, orc.SynthTridiagCtx(n, 1))
                want = OO.jacobian_oop(twin, x, fd, sparsity=(n, n, cp, rv), colorvec=cv, jac_prototype=("sparse", n, n),
                                       dir=dir, eps_override=list(cache._last_plan.eps()))
                assert_same_result(res, want, f"{devs} C2 {fd}: against the restatement")
            g.close()
            del single, res


def test_group_mirror_calls(pkg, fdist):
    """through the mirror, forward mode: 1 + C calls in all (f(x) once, at the root); central: 2C"""
    n = 12
    for kind in KINDS:
        for fd in ("forward", "central"):
            tk, lk, cv, C_ = _problem(pkg, kind, n)
            xd = torch.from_numpy(_x(n, seed=3)).cuda()
            g = _group(fdist, [0, 0, 0], kind, fd, tk)
            fs = [TorchF(f_nl) for _ in range(3)]
            g.run(fs, xd)
            torch.cuda.synchronize()
            assert sum(len(f.points) for f in fs) == (2 * C_ if fd == "central" else 1 + C_), (kind, fd)
            g.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_group_refusals(pkg, fdist):
    L = pkg._lib
    lib = L.lib()
    n = 10
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    cp, rv = tridiag_csc(n)
    xd = torch.from_numpy(_x(n)).cuda()
    J = torch.full((n, n), NAN, dtype=torch.float64, device="cuda")
    tf = TorchF(f_nl)
    addr, ctxs, keep = _trampolines(pkg, [tf, tf], n, [0, 0])
    devs = (C.c_int * 2)(0, 0)
    out = L.OopOut()
    out.J = J.data_ptr()
    oop = _abi_group(pkg, [0, 0], "csc_dense", n, cv, "forward")
    jac, hes = C.c_void_p(), C.c_void_p()
    o = pkg.api._opts(L.FDB_FORWARD, 0)
    L.check(lib.fdb_group_create_csc(C.byref(jac), 2, devs, n, n, cp.ctypes.data, rv.ctypes.data, L.FDB_J_DENSE, None,
                                     None, n, cv.ctypes.data, C.byref(o)))
    oh = pkg.api._opts(L.FDB_HCENTRAL, 0)
    L.check(lib.fdb_group_create_hessian(C.byref(hes), 2, devs, n, n, C.byref(oh)))
    try:
        st = lib.fdb_group_jacobian(oop, addr, ctxs, xd.data_ptr(), J.data_ptr(), None, None, NAN, NAN, 1.0, None)
        assert st == L.FDB_ERR_INVALID and b"fdb_group_jacobian_oop" in lib.fdb_last_error()
        st = lib.fdb_group_hessian(oop, addr, ctxs, xd.data_ptr(), J.data_ptr(), None, NAN, NAN, None)
        assert st == L.FDB_ERR_INVALID
        for g in (jac, hes):
            st = lib.fdb_group_jacobian_oop(g, addr, ctxs, xd.data_ptr(), C.byref(out), None, None, NAN, NAN, 1.0, None)
            assert st == L.FDB_ERR_INVALID and b"not an out-of-place group" in lib.fdb_last_error()
        torch.cuda.synchronize()
        assert len(tf.points) == 0 and torch.isnan(J).all(), "a refused call evaluates nothing and writes nothing"
    finally:
        for g in (oop, jac, hes):
            lib.fdb_group_destroy(g)
    # a sparse rank plan with world > 1 is refused by fdb_jacobian_oop: the group entry runs it
    for kind in ("csc_sparse", "sparse_proto"):
        p = _rank_plan(pkg, kind, n, cv if kind == "csc_sparse" else None, 1, 2, proto_cols=n)
        a, c, k = pkg.api._as_fn(tf, n, n, xd.device, 1, oop=True)
        E = 3 * n - 2 if kind == "csc_sparse" else n * n
        bufs = [torch.zeros(n + 1, dtype=torch.int64, device="cuda"), torch.zeros(E, dtype=torch.int64, device="cuda"),
                torch.zeros(E, dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")]
        so = L.OopOut()
        so.colptr, so.rowval, so.nzval, so.cap, so.nnz = bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), E, bufs[3].data_ptr()
        st = lib.fdb_jacobian_oop(p.handle, a, c, xd.data_ptr(), C.byref(so), None, None, NAN, NAN, 1.0, None)
        assert st == L.FDB_ERR_INVALID and b"fdb_group_jacobian_oop" in lib.fdb_last_error()
    assert len(tf.points) == 0
    # complex-step groups are not built
    oc = pkg.api._opts(L.FDB_COMPLEX, 0)
    g = C.c_void_p()
    L.check(lib.fdb_group_create_oop_csc(C.byref(g), 2, devs, n, n, cp.ctypes.data, rv.ctypes.data, cv.ctypes.data,
                                         L.FDB_OOP_DENSE, n, C.byref(oc)))
    try:
        st = lib.fdb_group_jacobian_oop(g, addr, ctxs, xd.data_ptr(), C.byref(out), None, None, NAN, NAN, 1.0, None)
        assert st == L.FDB_ERR_UNSUPPORTED
    finally:
        lib.fdb_group_destroy(g)
    torch.cuda.synchronize()
    assert len(tf.points) == 0 and torch.isnan(J).all()
