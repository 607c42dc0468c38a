"""What every plan creator reports, through the C ABI (run with -m gpu).

For one small problem of every creator this pins every fdb_plan_info field, fdb_plan_dense_range, the number of step
sizes fdb_plan_get_eps copies, and the plan's counters after one accepted call.  The values are literals: a change to
the plan's host-side bookkeeping that alters any reported value fails here.  FDB_SM_COUNT=1 and sizes far below the L2
thresholds keep device_bytes and the scatter strategy independent of the H100 model.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

NAN = float("nan")   # FDB_STEP_DEFAULT
CAP = 4096           # doubles / entries in every buffer handed to a call


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()._lib


@pytest.fixture(autouse=True)
def one_sm(monkeypatch):
    monkeypatch.setenv("FDB_SM_COUNT", "1")


def i64(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def band_csc(n, l, u, drop_first=False):
    """1-based CSC of the clipped band (l, u) of an n x n matrix; drop_first leaves out entry (1, 1)"""
    cols = [[r for r in range(max(0, c - u), min(n, c + l + 1))] for c in range(n)]
    if drop_first:
        cols[0] = cols[0][1:]
    colptr = i64(np.cumsum([1] + [len(c) for c in cols]))
    rowval = i64([r + 1 for c in cols for r in c])
    colidx = i64([j + 1 for j, c in enumerate(cols) for _ in c])
    return colptr, rowval, colidx


N = 8
CP, RV, CI = band_csc(N, 1, 1)                 # tridiagonal, 3 cyclic colours
CP5, RV5, _ = band_csc(N, 2, 2)                # pentadiagonal: a J pattern that holds the tridiagonal one
NL = 400                                        # > 1024 entries: one staged tile
CPL, RVL, _ = band_csc(NL, 1, 1)
CPD, RVD, _ = band_csc(NL, 1, 1, drop_first=True)
CV = i64(np.arange(N) % 3 + 1)
CVL = i64(np.arange(NL) % 3 + 1)
SLOTS = i64(np.arange(len(RV)) + 1)
BLOCKS = i64([4, 4])


def d(a):
    return a.ctypes.data


class Fn:
    """A Python f!: fx[r] = sin(x[r mod n]) (r + 1) + x[(r + 1) mod n]^2 / 2."""

    def __init__(self, L, m, n):
        self.L, self.m, self.n = L, max(m, 1), max(n, 1)
        self.ptr = L.FDB_FN(self._f)

    def _f(self, ctx, d_fx, d_x, batch, ldfx, ldx, stream):
        try:
            lib = self.L.lib()
            x = np.zeros((batch - 1) * ldx + self.n)
            fx = np.zeros((batch - 1) * ldfx + self.m)
            lib.fdb_memcpy_d2h(x.ctypes.data, d_x, x.nbytes, stream)
            lib.fdb_stream_sync(stream)
            r = np.arange(self.m)
            for b in range(batch):
                xb = x[b * ldx:b * ldx + self.n]
                fx[b * ldfx:b * ldfx + self.m] = np.sin(xb[r % self.n]) * (r + 1) + xb[(r + 1) % self.n] ** 2 / 2
            lib.fdb_memcpy_h2d(d_fx, fx.ctypes.data, fx.nbytes, stream)
            lib.fdb_stream_sync(stream)
            return 0
        except Exception:   # noqa: BLE001 — a C callback must not raise
            return 1


def opts(L, fdtype="FDB_FORWARD", **kw):
    o = L.PlanOpts()
    o.fdtype = getattr(L, fdtype)
    o.use_current_device = 1
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _csc(jkind, ldJ=0, n=N, cp=CP, rv=RV, cv=CV, j=None):
    return lambda L, lib, h, o: lib.fdb_plan_create_csc(
        h, n, n, d(cp), d(rv), getattr(L, jkind), d(j[0]) if j else None, d(j[1]) if j else None, ldJ, d(cv), o)


def _banded(jkind, ldJ):
    return lambda L, lib, h, o: lib.fdb_plan_create_banded(h, N, N, 1, 1, getattr(L, jkind), ldJ, d(CV), o)


# name -> (create(L, lib, handle_ref), plan options, the call it takes: "jacobian" | "oop" | "eps" | "jvp" | "hessian" |
# "derivative")
CASES = {
    "csc_fused": (_csc("FDB_J_CSC_NZVAL"), {}, "jacobian"),
    "csc_fused_central": (_csc("FDB_J_CSC_NZVAL"), {"fdtype": "FDB_CENTRAL"}, "jacobian"),
    "csc_staged": (_csc("FDB_J_CSC_NZVAL", n=NL, cp=CPD, rv=RVD, cv=CVL), {}, "jacobian"),
    "csc_band_form": (_csc("FDB_J_CSC_NZVAL", n=NL, cp=CPL, rv=RVL, cv=CVL), {}, "jacobian"),
    "csc_lists": (_csc("FDB_J_CSC_NZVAL"), {"strategy": 2, "scratch_bytes": 8 * 8}, "jacobian"),
    "csc_lists_resident": (_csc("FDB_J_CSC_NZVAL"), {"strategy": 3}, "jacobian"),
    "csc_dense_j": (_csc("FDB_J_DENSE", ldJ=N + 2), {}, "jacobian"),
    "csc_other_j": (_csc("FDB_J_CSC_NZVAL", j=(CP5, RV5)), {}, "jacobian"),
    "coo": (lambda L, lib, h, o: lib.fdb_plan_create_coo(h, N, N, len(RV), d(RV), d(CI), L.FDB_J_SLOTS, d(SLOTS),
                                                         len(RV), d(CV), o), {}, "jacobian"),
    "banded_band": (_banded("FDB_J_BAND", 3), {}, "jacobian"),
    "banded_dense": (_banded("FDB_J_DENSE", N), {}, "jacobian"),
    "banded_diagonals": (_banded("FDB_J_DIAGONALS", 3 * N - 2), {}, "jacobian"),
    "block_banded": (lambda L, lib, h, o: lib.fdb_plan_create_block_banded(h, 2, d(BLOCKS), 1, 1, 1, 1, 9 * N, None, o),
                     {}, "jacobian"),
    "dense": (lambda L, lib, h, o: lib.fdb_plan_create_dense(h, N, N, N, o), {}, "jacobian"),
    "dense_central": (lambda L, lib, h, o: lib.fdb_plan_create_dense(h, N, N, N, o), {"fdtype": "FDB_CENTRAL"},
                      "jacobian"),
    "dense_colorvec": (lambda L, lib, h, o: lib.fdb_plan_create_dense_colorvec(h, N, N, N, d(CV), o), {}, "jacobian"),
    "dense_rank": (lambda L, lib, h, o: lib.fdb_plan_create_dense(h, N, N, N, o), {"world": 3, "rank": 1}, "jacobian"),
    "eps": (lambda L, lib, h, o: lib.fdb_eps_plan_create(h, N, d(CV), o), {}, "eps"),
    "jvp": (lambda L, lib, h, o: lib.fdb_jvp_plan_create(h, N, N, o), {}, "jvp"),
    "hessian": (lambda L, lib, h, o: lib.fdb_hessian_plan_create(h, N, N, o), {"fdtype": "FDB_HCENTRAL"}, "hessian"),
    "hessian_rank": (lambda L, lib, h, o: lib.fdb_hessian_plan_create(h, N, N, o),
                     {"fdtype": "FDB_HCENTRAL", "world": 2, "rank": 1}, "hessian"),
    "derivative": (lambda L, lib, h, o: lib.fdb_derivative_plan_create(h, N, o), {}, "derivative"),
    "derivative_central": (lambda L, lib, h, o: lib.fdb_derivative_plan_create(h, N, o),
                           {"fdtype": "FDB_CENTRAL", "max_batch": 2}, "derivative"),
    "scalar_gradient": (lambda L, lib, h, o: lib.fdb_scalar_gradient_plan_create(h, N, o), {}, "derivative"),
    "oop_csc_dense": (lambda L, lib, h, o: lib.fdb_oop_plan_create_csc(h, N, N, d(CP), d(RV), d(CV), L.FDB_OOP_DENSE, N,
                                                                       o), {}, "oop"),
    "oop_csc_sparse": (lambda L, lib, h, o: lib.fdb_oop_plan_create_csc(h, N, N, d(CP), d(RV), d(CV), L.FDB_OOP_SPARSE,
                                                                        0, o), {}, "oop"),
    "oop_banded_dense": (lambda L, lib, h, o: lib.fdb_oop_plan_create_banded(h, N, N, 1, 1, d(CV), L.FDB_OOP_DENSE, N,
                                                                             o), {}, "oop"),
    "oop_banded_sparse": (lambda L, lib, h, o: lib.fdb_oop_plan_create_banded(h, N, N, 1, 1, d(CV), L.FDB_OOP_SPARSE, 0,
                                                                              o), {}, "oop"),
    "oop_dense_raw": (lambda L, lib, h, o: lib.fdb_oop_plan_create_dense(h, N, N, d(CV), 0, L.FDB_OOP_RAW, N, o), {},
                      "oop"),
    "oop_dense_dense": (lambda L, lib, h, o: lib.fdb_oop_plan_create_dense(h, N, N, d(CV), N, L.FDB_OOP_DENSE, N, o),
                        {}, "oop"),
    "oop_dense_sparse": (lambda L, lib, h, o: lib.fdb_oop_plan_create_dense(h, N, N, d(CV), N, L.FDB_OOP_SPARSE, 0, o),
                         {}, "oop"),
}


def plan_state(L, name):
    """(fdb_plan_info, fdb_plan_dense_range, fdb_plan_get_eps length, counters after one call) of case `name`"""
    create, kw, kind = CASES[name]
    lib = L.lib()
    h = C.c_void_p()
    o = opts(L, **kw)
    L.check(create(L, lib, C.byref(h), C.byref(o)))
    try:
        i = L.PlanInfo()
        L.check(lib.fdb_plan_info(h, C.byref(i)))
        info = i.as_dict()
        f = Fn(L, info["m"], info["n"])
        fp = C.cast(f.ptr, C.c_void_p)
        dev = torch.device("cuda:0")
        x = 0.3 + 0.1 * torch.arange(CAP, dtype=torch.float64, device=dev)
        v = torch.ones(CAP, dtype=torch.float64, device=dev)
        J, fx, eps, nzval = (torch.zeros(CAP, dtype=torch.float64, device=dev) for _ in range(4))
        colptr, rowval, nnz = (torch.zeros(CAP, dtype=torch.int64, device=dev) for _ in range(3))
        out = L.OopOut(J.data_ptr(), colptr.data_ptr(), rowval.data_ptr(), nzval.data_ptr(), CAP, nnz.data_ptr())
        p = lambda t: t.data_ptr()   # noqa: E731
        L.check({
            "jacobian": lambda: lib.fdb_jacobian(h, fp, None, p(x), p(J), p(fx), None, NAN, NAN, 1.0, None),
            "oop": lambda: lib.fdb_jacobian_oop(h, fp, None, p(x), C.byref(out), p(fx), None, NAN, NAN, 1.0, None),
            "eps": lambda: lib.fdb_color_eps(h, p(x), NAN, NAN, 1.0, p(eps), None),
            "jvp": lambda: lib.fdb_jvp(h, fp, None, p(J), p(x), p(v), None, None, None, NAN, NAN, 1.0, None),
            "hessian": lambda: lib.fdb_hessian(h, fp, None, p(x), p(J), p(fx), NAN, NAN, None),
            "derivative": lambda: lib.fdb_derivative(h, fp, None, p(J), p(x), None, NAN, NAN, 1.0, None),
        }[kind]())
        torch.cuda.synchronize()
        b, e = C.c_int64(), C.c_int64()
        L.check(lib.fdb_plan_dense_range(h, C.byref(b), C.byref(e)))
        eps_len = None   # derivative plans keep no step sizes
        if kind != "derivative":
            heps = np.full(CAP, np.nan)
            L.check(lib.fdb_plan_get_eps(h, heps.ctypes.data_as(C.POINTER(C.c_double)), CAP, None))
            eps_len = int(np.count_nonzero(~np.isnan(heps)))
        c = L.Counters()
        L.check(lib.fdb_plan_counters(h, C.byref(c)))
        return {"info": info, "dense_range": (b.value, e.value), "eps_len": eps_len, "counters": c.as_dict()}
    finally:
        lib.fdb_plan_destroy(h)


# name -> (fdb_plan_info_t fields in INFO order, fdb_plan_dense_range, fdb_plan_get_eps length (None: refused),
#          fdb_counters_t fields in COUNTERS order)
INFO = ("m", "n", "n_entries", "j_len", "n_colors", "n_local_colors", "n_groups", "slabs", "fcalls_per_jacobian",
        "device_bytes", "fdtype", "jkind", "sp_kind", "color_bits", "alg_bytes_scatter", "strategy", "lanes",
        "mean_row_jump", "moved_bytes_scatter", "staged", "lists_resident")
COUNTERS = ("jacobians", "f_points", "f_invocations", "kernel_launches", "scatter_launches")
EXPECTED = {
    "csc_fused": ((8, 8, 22, 22, 3, 3, 1, 3, 4, 802, 0, 0, 1, 8, 840, 0, 4, 1.0, 526, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "csc_fused_central": ((8, 8, 22, 22, 3, 3, 1, 3, 6, 1186, 1, 0, 1, 8, 840, 0, 4, 1.0, 638, 0, 0),
        (0, 0), 3, (1, 6, 6, 3, 1)),
    "csc_staged": ((400, 400, 1197, 1197, 3, 3, 1, 3, 4, 34217, 0, 0, 1, 8, 44712, 0, 4, 1.0, 24770, 1, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "csc_band_form": ((400, 400, 1198, 1198, 3, 3, 1, 3, 4, 34222, 0, 0, 1, 8, 44744, 0, 4, 1.0, 22384, 1, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "csc_lists": ((8, 8, 22, 22, 3, 3, 3, 1, 4, 930, 0, 0, 1, 8, 840, 1, 4, 1.0, 1032, 0, 0),
        (0, 0), 3, (1, 4, 4, 8, 3)),
    "csc_lists_resident": ((8, 8, 22, 22, 3, 3, 1, 3, 4, 1010, 0, 0, 1, 8, 840, 1, 4, 1.0, 592, 0, 1),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "csc_dense_j": ((8, 8, 22, 80, 3, 3, 1, 3, 4, 978, 0, 1, 1, 8, 840, 0, 4, 1.0, 702, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "csc_other_j": ((8, 8, 22, 34, 3, 3, 1, 3, 4, 978, 0, 0, 1, 8, 840, 0, 4, 1.0, 702, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "coo": ((8, 8, 22, 22, 3, 3, 1, 3, 4, 910, 0, 3, 3, 8, 840, 0, 1, 0.0, 702, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "banded_band": ((8, 8, 22, 24, 3, 3, 1, 3, 4, 608, 0, 2, 4, 8, 560, 0, 1, 0.0, 560, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "banded_dense": ((8, 8, 22, 64, 3, 3, 1, 3, 4, 608, 0, 1, 4, 8, 560, 0, 1, 0.0, 560, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "banded_diagonals": ((8, 8, 22, 22, 3, 3, 1, 3, 4, 608, 0, 5, 4, 8, 560, 0, 1, 0.0, 560, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 1)),
    "block_banded": ((8, 8, 40, 72, 8, 8, 1, 8, 9, 1124, 0, 4, 9, 8, 1600, 0, 1, 0.0, 1600, 0, 0),
        (0, 0), 8, (1, 9, 9, 4, 1)),
    "dense": ((8, 8, 64, 64, 8, 8, 8, 1, 9, 256, 0, 1, 0, 8, 1536, 0, 1, 0.0, 1536, 0, 0),
        (0, 8), 8, (1, 9, 9, 18, 8)),
    "dense_central": ((8, 8, 64, 64, 8, 8, 8, 1, 16, 320, 1, 1, 0, 8, 1536, 0, 1, 0.0, 1536, 0, 0),
        (0, 8), 8, (1, 16, 16, 26, 8)),
    "dense_colorvec": ((8, 8, 24, 24, 8, 3, 3, 1, 4, 216, 0, 1, 0, 8, 576, 0, 1, 0.0, 576, 0, 0),
        (0, 3), 3, (1, 4, 4, 8, 3)),
    "dense_rank": ((8, 8, 24, 24, 8, 3, 3, 1, 4, 216, 0, 1, 0, 8, 576, 0, 1, 0.0, 576, 0, 0),
        (3, 6), 3, (1, 4, 4, 8, 3)),
    "eps": ((0, 8, 0, 0, 3, 0, 0, 0, 1, 136, 0, 0, 6, 8, 0, 0, 1, 0.0, 0, 0, 0),
        (0, 0), 3, (0, 0, 0, 1, 0)),
    "jvp": ((8, 8, 0, 0, 1, 0, 0, 0, 1, 184, 0, 0, 5, 8, 384, 0, 1, 0.0, 384, 0, 0),
        (0, 0), 1, (1, 2, 2, 3, 0)),
    "hessian": ((1, 8, 64, 64, 8, 8, 1, 1, 129, 1160, 3, 1, 7, 8, 5448, 0, 1, 0.0, 5448, 0, 0),
        (0, 8), 8, (1, 129, 129, 132, 1)),
    "hessian_rank": ((1, 8, 36, 64, 8, 6, 1, 1, 73, 712, 3, 1, 7, 8, 3048, 0, 1, 0.0, 3048, 0, 0),
        (2, 8), 6, (1, 73, 73, 76, 1)),
    "derivative": ((8, 8, 8, 8, 0, 0, 0, 0, 2, 256, 0, 1, 8, 8, 384, 0, 1, 0.0, 384, 0, 0),
        (0, 0), None, (1, 2, 2, 2, 1)),
    "derivative_central": ((8, 8, 8, 8, 0, 0, 0, 0, 2, 256, 1, 1, 8, 8, 448, 0, 1, 0.0, 448, 0, 0),
        (0, 0), None, (1, 2, 1, 2, 1)),
    "scalar_gradient": ((8, 1, 8, 8, 0, 0, 0, 0, 2, 160, 0, 1, 8, 8, 208, 0, 1, 0.0, 208, 0, 0),
        (0, 0), None, (1, 2, 2, 2, 1)),
    "oop_csc_dense": ((8, 8, 22, 64, 3, 3, 1, 3, 4, 978, 0, 1, 1, 8, 840, 0, 4, 1.0, 702, 0, 0),
        (0, 0), 3, (1, 4, 4, 4, 1)),
    "oop_csc_sparse": ((8, 8, 22, 22, 3, 3, 1, 3, 4, 998, 0, 0, 1, 8, 840, 0, 4, 1.0, 526, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 0)),
    "oop_banded_dense": ((8, 8, 22, 64, 3, 3, 1, 3, 4, 608, 0, 1, 4, 8, 560, 0, 1, 0.0, 560, 0, 0),
        (0, 0), 3, (1, 4, 4, 4, 1)),
    "oop_banded_sparse": ((8, 8, 22, 24, 3, 3, 1, 3, 4, 640, 0, 2, 4, 8, 560, 0, 1, 0.0, 560, 0, 0),
        (0, 0), 3, (1, 4, 4, 3, 0)),
    "oop_dense_raw": ((8, 8, 24, 24, 8, 3, 3, 1, 4, 216, 0, 1, 0, 8, 576, 0, 1, 0.0, 576, 0, 0),
        (0, 3), 3, (1, 4, 4, 8, 3)),
    "oop_dense_dense": ((8, 8, 24, 24, 8, 3, 3, 1, 4, 216, 0, 1, 0, 8, 576, 0, 1, 0.0, 576, 0, 0),
        (0, 3), 3, (1, 4, 4, 9, 3)),
    "oop_dense_sparse": ((8, 8, 24, 24, 8, 3, 3, 1, 4, 424, 0, 1, 0, 8, 576, 0, 1, 0.0, 576, 0, 0),
        (0, 3), 3, (1, 4, 4, 9, 3)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_plan_state(L, name):
    got = plan_state(L, name)
    info, dense_range, eps_len, counters = EXPECTED[name]
    assert got["info"] == dict(zip(INFO, info))
    assert got["dense_range"] == dense_range
    assert got["eps_len"] == eps_len
    assert got["counters"] == dict(zip(COUNTERS, counters))
