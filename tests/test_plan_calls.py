"""Which calls each plan takes, through the C ABI (run with -m gpu).

One plan of every kind, in every fdtype its creator accepts, meets every compute and query call whose acceptance depends
on the plan, always with valid buffers.  Each (plan, call) cell must give the status and fdb_last_error() text of the
table below (include/fdjac_b200.h states the same rule).  A refused call must not call f and must leave the plan's
counters as they were; the call the plan does take must then return exactly what it returns on a freshly built plan.
The group calls are checked the same way on groups over devices [0, 0].
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N = 8                                  # m = n = 8: a tridiagonal pattern, 3 cyclic colours
NAN = float("nan")                     # FDB_STEP_DEFAULT
CAP = 1024                             # doubles / entries in every buffer handed to a call


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()._lib


def i64(v):
    return np.ascontiguousarray(v, dtype=np.int64)


ROWS = [r for c in range(N) for r in range(max(0, c - 1), min(N, c + 2))]
COLPTR = i64(np.cumsum([1] + [min(N, c + 2) - max(0, c - 1) for c in range(N)]))
ROWVAL = i64(np.array(ROWS) + 1)
COLS = i64([c + 1 for c in range(N) for _ in range(max(0, c - 1), min(N, c + 2))])
CV = i64(np.arange(N) % 3 + 1)
SLOTS = i64(np.arange(len(ROWVAL)) + 1)
BLOCKS = i64([4, 4])


class Fn:
    """A Python f! that counts its calls: fx[r] = sin(x[r mod n]) (r + 1) + x[(r + 1) mod n]^2 / 2, real or complex128."""

    def __init__(self, L, m, n, cplx):
        self.L, self.m, self.n, self.cplx, self.calls = L, m, n, cplx, 0
        self.ptr = L.FDB_FN(self._f)

    def _f(self, ctx, d_fx, d_x, batch, ldfx, ldx, stream):
        try:
            self.calls += 1
            dt = np.complex128 if self.cplx else np.float64
            lib = self.L.lib()
            x = np.zeros((batch - 1) * ldx + self.n, dtype=dt)
            fx = np.zeros((batch - 1) * ldfx + self.m, dtype=dt)
            lib.fdb_memcpy_d2h(x.ctypes.data, d_x, x.nbytes, stream)
            lib.fdb_memcpy_d2h(fx.ctypes.data, d_fx, fx.nbytes, stream)
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


# ------------------------------------------------------------------------------------------------ plans
# name -> (class, fdtypes, create(L, handle_ref, opts)); the class picks the row of the table
PLANS = {
    "csc_nzval": ("csc", "fcx", lambda L, h, o: L.lib().fdb_plan_create_csc(
        h, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, L.FDB_J_CSC_NZVAL, None, None, 0, CV.ctypes.data, o)),
    "csc_dense": ("csc", "fcx", lambda L, h, o: L.lib().fdb_plan_create_csc(
        h, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, L.FDB_J_DENSE, None, None, N, CV.ctypes.data, o)),
    "coo_slots": ("csc", "fcx", lambda L, h, o: L.lib().fdb_plan_create_coo(
        h, N, N, len(ROWVAL), ROWVAL.ctypes.data, COLS.ctypes.data, L.FDB_J_SLOTS, SLOTS.ctypes.data, len(ROWVAL),
        CV.ctypes.data, o)),
    "banded_band": ("band", "fcx", lambda L, h, o: L.lib().fdb_plan_create_banded(
        h, N, N, 1, 1, L.FDB_J_BAND, 3, CV.ctypes.data, o)),
    "banded_diagonals": ("band", "fcx", lambda L, h, o: L.lib().fdb_plan_create_banded(
        h, N, N, 1, 1, L.FDB_J_DIAGONALS, 3 * N - 2, CV.ctypes.data, o)),
    "block_banded": ("band", "fcx", lambda L, h, o: L.lib().fdb_plan_create_block_banded(
        h, 2, BLOCKS.ctypes.data, 1, 1, 1, 1, 9 * N, None, o)),
    "dense": ("dense", "fcx", lambda L, h, o: L.lib().fdb_plan_create_dense(h, N, N, N, o)),
    "dense_colorvec": ("dense", "fcx", lambda L, h, o: L.lib().fdb_plan_create_dense_colorvec(
        h, N, N, N, CV.ctypes.data, o)),
    "eps": ("eps", "fcx", lambda L, h, o: L.lib().fdb_eps_plan_create(h, N, CV.ctypes.data, o)),
    "jvp": ("jvp", "fc", lambda L, h, o: L.lib().fdb_jvp_plan_create(h, N, N, o)),
    "hessian": ("hess", "h", lambda L, h, o: L.lib().fdb_hessian_plan_create(h, N, N, o)),
    "derivative": ("deriv", "fcx", lambda L, h, o: L.lib().fdb_derivative_plan_create(h, N, o)),
    "scalar_gradient": ("deriv", "fcx", lambda L, h, o: L.lib().fdb_scalar_gradient_plan_create(h, N, o)),
    "oop_csc_dense": ("oop_csc", "fcx", lambda L, h, o: L.lib().fdb_oop_plan_create_csc(
        h, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, CV.ctypes.data, L.FDB_OOP_DENSE, N, o)),
    "oop_csc_sparse": ("oop_csc", "fcx", lambda L, h, o: L.lib().fdb_oop_plan_create_csc(
        h, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, CV.ctypes.data, L.FDB_OOP_SPARSE, 0, o)),
    "oop_dense_raw": ("oop_dense", "fcx", lambda L, h, o: L.lib().fdb_oop_plan_create_dense(
        h, N, N, CV.ctypes.data, 0, L.FDB_OOP_RAW, N, o)),
    "oop_dense_dense": ("oop_dense", "fcx", lambda L, h, o: L.lib().fdb_oop_plan_create_dense(
        h, N, N, CV.ctypes.data, N, L.FDB_OOP_DENSE, N, o)),
    "oop_dense_sparse": ("oop_dense", "fcx", lambda L, h, o: L.lib().fdb_oop_plan_create_dense(
        h, N, N, CV.ctypes.data, N, L.FDB_OOP_SPARSE, 0, o)),
}
FDTYPE = {"f": "FDB_FORWARD", "c": "FDB_CENTRAL", "x": "FDB_COMPLEX", "h": "FDB_HCENTRAL"}
CASES = [(p, t) for p, (_, ts, _) in PLANS.items() for t in ts]


def make_plan(L, name, t):
    o = L.PlanOpts()
    o.fdtype = getattr(L, FDTYPE[t])
    o.use_current_device = 1
    h = C.c_void_p()
    L.check(PLANS[name][2](L, C.byref(h), C.byref(o)))
    return h


def info(L, h):
    i = L.PlanInfo()
    L.check(L.lib().fdb_plan_info(h, C.byref(i)))
    return i


def counters(L, h):
    c = L.Counters()
    L.check(L.lib().fdb_plan_counters(h, C.byref(c)))
    return c.as_dict()


# ------------------------------------------------------------------------------------------------ the expected table
# call -> {plan class: (outcome on a real plan, outcome on a complex plan)}; None = accepted, else (status, message)
def bad(msg, status="INVALID"):
    return (status, msg)


def both(o):
    return (o, o)


JAC_KIND = {
    "eps": both(bad("this is a step-size plan: call fdb_color_eps")),
    "jvp": both(bad("this is a JVP plan: call fdb_jvp")),
    "hess": both(bad("this is a Hessian plan: call fdb_hessian")),
    "deriv": both(bad("this is a derivative plan: call fdb_derivative")),
    "oop_csc": both(bad("this is an out-of-place plan: call fdb_jacobian_oop")),
    "oop_dense": both(bad("this is an out-of-place plan: call fdb_jacobian_oop")),
}
CPLX_J = bad("this plan is a complex-step plan: call fdb_jacobian_complex with a complex128 callback")
NEED_CJ = bad("fdb_jacobian_complex needs a plan created with fdtype = FDB_COMPLEX")
CPLX_OOP = bad("this plan is a complex-step plan: call fdb_jacobian_oop_complex with a complex128 callback")
NEED_COOP = bad("fdb_jacobian_oop_complex needs a plan created with fdtype = FDB_COMPLEX")
NOT_OOP = bad("not an out-of-place plan (fdb_oop_plan_create_csc / _dense)")
NOT_COLOURED = bad("fdb_color_eps needs a coloured plan")
NOT_EXT = bad("external step sizes apply to coloured Jacobian plans")
NO_PEERS = bad("peer stores are implemented for the entry-driven (CSC / COO) scatters", "UNSUPPORTED")
BY_RANGE = bad("dense plans partition columns by range")
NOT_JVP = bad("not a JVP plan (fdb_jvp_plan_create)")
NOT_HESS = bad("not a Hessian plan (fdb_hessian_plan_create)")
NOT_DERIV = bad("not a derivative plan (fdb_derivative_plan_create / fdb_scalar_gradient_plan_create)")
CPLX_D = bad("this plan is a complex-step plan: call fdb_derivative_complex with a complex128 callback")
NEED_CD = bad("fdb_derivative_complex needs a derivative plan created with fdtype = FDB_COMPLEX")
ALL = ("csc", "band", "dense", "eps", "jvp", "hess", "deriv", "oop_csc", "oop_dense")

TABLE = {
    "jacobian": {"csc": (None, CPLX_J), "band": (None, CPLX_J), "dense": (None, CPLX_J), **JAC_KIND},
    "jacobian_complex": {"csc": (NEED_CJ, None), "band": (NEED_CJ, None), "dense": (NEED_CJ, None),
                         **{k: (NEED_CJ, v[1]) for k, v in JAC_KIND.items()}},
    "jacobian_oop": {**{k: (NOT_OOP, CPLX_OOP) for k in ALL}, "oop_csc": (None, CPLX_OOP), "oop_dense": (None, CPLX_OOP)},
    "jacobian_oop_complex": {**{k: (NEED_COOP, NOT_OOP) for k in ALL}, "oop_csc": (NEED_COOP, None),
                             "oop_dense": (NEED_COOP, None)},
    "color_eps": {**{k: both(NOT_COLOURED) for k in ALL}, "csc": both(None), "band": both(None), "eps": both(None),
                  "oop_csc": both(None)},
    "set_external_eps": {**{k: both(NOT_EXT) for k in ALL}, "csc": both(None), "band": both(None), "oop_csc": both(None)},
    "set_peers": {**{k: both(NO_PEERS) for k in ALL}, "csc": both(None), "eps": both(None), "jvp": both(None),
                  "oop_csc": both(None)},
    "color_owner": {**{k: both(None) for k in ALL}, "dense": both(BY_RANGE), "hess": both(BY_RANGE),
                    "oop_dense": both(BY_RANGE), "deriv": both(bad("derivative plans have no colours"))},
    "get_eps": {**{k: both(None) for k in ALL},
                "deriv": both(bad("derivative plans keep no step sizes (the quotient pass recomputes them)"))},
    "jvp": {**{k: both(NOT_JVP) for k in ALL}, "jvp": both(None)},
    "jvp_oop": {**{k: both(NOT_JVP) for k in ALL}, "jvp": both(None)},
    "hessian": {**{k: both(NOT_HESS) for k in ALL}, "hess": both(None)},
    "derivative": {**{k: both(NOT_DERIV) for k in ALL}, "deriv": (None, CPLX_D)},
    "derivative_complex": {**{k: both(NEED_CD) for k in ALL}, "deriv": (NEED_CD, None)},
}
TABLE["jacobian_host"] = TABLE["jacobian"]


def expected(call, name, t):
    return TABLE[call][PLANS[name][0]][1 if t == "x" else 0]


# ------------------------------------------------------------------------------------------------ the calls
class Bufs:
    """Valid device and host buffers for any call on an 8 x 8 problem."""

    def __init__(self, L):
        dev = torch.device("cuda:0")
        z = lambda dt=torch.float64: torch.zeros(CAP, dtype=dt, device=dev)   # noqa: E731
        self.x = z()
        self.x[:N] = 0.3 + 0.1 * torch.arange(N, dtype=torch.float64, device=dev)
        self.v = z()
        self.v[:N] = 1.0
        self.J, self.fx, self.eps, self.nzval = z(), z(), z(), z()
        self.colptr, self.rowval, self.nnz = z(torch.int64), z(torch.int64), z(torch.int64)
        self.out = L.OopOut(self.J.data_ptr(), self.colptr.data_ptr(), self.rowval.data_ptr(), self.nzval.data_ptr(),
                            CAP, self.nnz.data_ptr())
        self.hx = self.x.cpu().numpy().copy()
        self.hJ, self.hfx = np.zeros(CAP), np.zeros(CAP)
        self.owner = np.zeros(CAP, dtype=np.int32)
        self.heps = np.zeros(CAP)
        self.peers = (C.c_void_p * 1)()

    def result(self):
        torch.cuda.synchronize()
        return np.concatenate([t.cpu().numpy().view(np.int64) for t in
                               (self.J, self.fx, self.eps, self.nzval, self.colptr, self.rowval, self.nnz)]
                              + [self.hJ.view(np.int64), self.heps.view(np.int64)])


def call(L, name, h, f, b):
    lib, d = L.lib(), lambda t: t.data_ptr()   # noqa: E731
    fp = C.cast(f.ptr, C.c_void_p)
    return {
        "jacobian": lambda: lib.fdb_jacobian(h, fp, None, d(b.x), d(b.J), d(b.fx), None, NAN, NAN, 1.0, None),
        "jacobian_complex": lambda: lib.fdb_jacobian_complex(h, fp, None, d(b.x), d(b.J), None),
        "jacobian_host": lambda: lib.fdb_jacobian_host(h, fp, None, b.hx.ctypes.data, b.hJ.ctypes.data,
                                                       b.hfx.ctypes.data, None, NAN, NAN, 1.0),
        "jacobian_oop": lambda: lib.fdb_jacobian_oop(h, fp, None, d(b.x), C.byref(b.out), d(b.fx), None, NAN, NAN, 1.0,
                                                     None),
        "jacobian_oop_complex": lambda: lib.fdb_jacobian_oop_complex(h, fp, None, d(b.x), C.byref(b.out), None),
        "color_eps": lambda: lib.fdb_color_eps(h, d(b.x), NAN, NAN, 1.0, d(b.eps), None),
        "set_external_eps": lambda: lib.fdb_plan_set_external_eps(h, d(b.eps)),
        "set_peers": lambda: lib.fdb_plan_set_peers(h, 0, b.peers),
        "color_owner": lambda: lib.fdb_plan_color_owner(h, b.owner.ctypes.data_as(C.POINTER(C.c_int32)), CAP),
        "get_eps": lambda: lib.fdb_plan_get_eps(h, b.heps.ctypes.data_as(C.POINTER(C.c_double)), CAP, None),
        "jvp": lambda: lib.fdb_jvp(h, fp, None, d(b.J), d(b.x), d(b.v), None, None, None, NAN, NAN, 1.0, None),
        "jvp_oop": lambda: lib.fdb_jvp_oop(h, fp, None, d(b.J), d(b.x), d(b.v), None, None, None, NAN, NAN, 1.0, None),
        "hessian": lambda: lib.fdb_hessian(h, fp, None, d(b.x), d(b.J), d(b.fx), NAN, NAN, None),
        "derivative": lambda: lib.fdb_derivative(h, fp, None, d(b.J), d(b.x), None, NAN, NAN, 1.0, None),
        "derivative_complex": lambda: lib.fdb_derivative_complex(h, fp, None, d(b.J), d(b.x), None),
    }[name]()


CALLS = list(TABLE)


def accepted_call(name, t):
    """the computing call plan `name` of fdtype t takes"""
    for c in ("jacobian", "jacobian_complex", "jacobian_oop", "jacobian_oop_complex", "jvp", "hessian", "derivative",
              "derivative_complex", "color_eps"):
        if expected(c, name, t) is None:
            return c
    raise AssertionError(name)


def fn_for(L, h, t):
    i = info(L, h)
    return Fn(L, max(i.m, 1), max(i.n, 1), t == "x")


def run_accepted(L, name, t, h):
    b = Bufs(L)
    c = accepted_call(name, t)
    L.check(call(L, c, h, fn_for(L, h, t), b))
    return b.result()


_fresh = {}


def fresh_result(L, name, t):
    if (name, t) not in _fresh:
        h = make_plan(L, name, t)
        try:
            _fresh[name, t] = run_accepted(L, name, t, h)
        finally:
            L.lib().fdb_plan_destroy(h)
    return _fresh[name, t]


@pytest.mark.parametrize("name,t", CASES)
@pytest.mark.parametrize("c", CALLS)
def test_call_on_plan(L, c, name, t):
    want = expected(c, name, t)
    h = make_plan(L, name, t)
    try:
        f = fn_for(L, h, t)
        before = counters(L, h)
        st = call(L, c, h, f, Bufs(L))
        torch.cuda.synchronize()
        msg = L.lib().fdb_last_error().decode()
        if want is None:
            assert st == L.FDB_OK, f"{c} on {name}/{t}: refused with {st}: {msg}"
            return
        status, text = want
        assert (st, msg) == (getattr(L, f"FDB_ERR_{status}"), text)
        assert f.calls == 0, f"{c} on {name}/{t} called f although it refused the plan"
        assert counters(L, h) == before
        # the plan still computes exactly what a fresh one does
        assert np.array_equal(run_accepted(L, name, t, h), fresh_result(L, name, t))
    finally:
        L.lib().fdb_plan_destroy(h)


HOST_REFUSED = [(n, t) for n, t in CASES if expected("jacobian_host", n, t) is not None]


@pytest.mark.parametrize("name,t", HOST_REFUSED)
def test_refused_host_call_allocates_nothing(L, name, t):
    """fdb_jacobian_host refuses the plan before it creates its stream and host-path buffers."""
    h = make_plan(L, name, t)
    try:
        before = info(L, h).device_bytes
        assert call(L, "jacobian_host", h, fn_for(L, h, t), Bufs(L)) != L.FDB_OK
        assert info(L, h).device_bytes == before
    finally:
        L.lib().fdb_plan_destroy(h)


# ------------------------------------------------------------------------------------------------ groups over [0, 0]
GROUPS = {
    "csc": ("csc", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_csc(
        h, 2, d, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, L.FDB_J_CSC_NZVAL, None, None, 0, CV.ctypes.data, o)),
    "banded": ("band", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_banded(
        h, 2, d, N, N, 1, 1, L.FDB_J_BAND, 3, CV.ctypes.data, o)),
    "dense": ("dense", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_dense(h, 2, d, N, N, N, o)),
    "block_banded": ("band", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_block_banded(
        h, 2, d, 2, BLOCKS.ctypes.data, 1, 1, 1, 1, 9 * N, None, o)),
    "hessian": ("hess", "h", lambda L, h, d, o: L.lib().fdb_group_create_hessian(h, 2, d, N, N, o)),
    "oop_csc": ("oop", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_oop_csc(
        h, 2, d, N, N, COLPTR.ctypes.data, ROWVAL.ctypes.data, CV.ctypes.data, L.FDB_OOP_DENSE, N, o)),
    "oop_dense": ("oop", "fcx", lambda L, h, d, o: L.lib().fdb_group_create_oop_dense(
        h, 2, d, N, N, CV.ctypes.data, N, L.FDB_OOP_DENSE, N, o)),
}
GROUPS_UNSUP = bad("groups run forward / central plans", "UNSUPPORTED")
NOT_OOP_GROUP = bad("not an out-of-place group (fdb_group_create_oop_csc / _dense)")
NOT_HESS_GROUP = bad("not a Hessian group (fdb_group_create_hessian)")
GROUP_TABLE = {
    "group_jacobian": {"csc": (None, GROUPS_UNSUP), "band": (None, GROUPS_UNSUP), "dense": (None, GROUPS_UNSUP),
                       "hess": both(bad("this is a Hessian group: call fdb_group_hessian")),
                       "oop": both(bad("this is an out-of-place group: call fdb_group_jacobian_oop"))},
    "group_jacobian_oop": {"csc": both(NOT_OOP_GROUP), "band": both(NOT_OOP_GROUP), "dense": both(NOT_OOP_GROUP),
                           "hess": both(NOT_OOP_GROUP), "oop": (None, GROUPS_UNSUP)},
    "group_hessian": {"csc": both(NOT_HESS_GROUP), "band": both(NOT_HESS_GROUP), "dense": both(NOT_HESS_GROUP),
                      "hess": both(None), "oop": both(NOT_HESS_GROUP)},
}
GROUP_CASES = [(g, t) for g, (_, ts, _) in GROUPS.items() for t in ts]


def make_group(L, name, t):
    o = L.PlanOpts()
    o.fdtype = getattr(L, FDTYPE[t])
    devs = (C.c_int * 2)(0, 0)
    h = C.c_void_p()
    L.check(GROUPS[name][2](L, C.byref(h), devs, C.byref(o)))
    return h


def group_call(L, c, g, f, b):
    lib, d = L.lib(), lambda t: t.data_ptr()   # noqa: E731
    fp, ctx = C.cast(f.ptr, C.c_void_p), (C.c_void_p * 2)()
    return {
        "group_jacobian": lambda: lib.fdb_group_jacobian(g, fp, ctx, d(b.x), d(b.J), d(b.fx), None, NAN, NAN, 1.0, None),
        "group_jacobian_oop": lambda: lib.fdb_group_jacobian_oop(g, fp, ctx, d(b.x), C.byref(b.out), d(b.fx), None, NAN,
                                                                 NAN, 1.0, None),
        "group_hessian": lambda: lib.fdb_group_hessian(g, fp, ctx, d(b.x), d(b.J), d(b.fx), NAN, NAN, None),
    }[c]()


def group_counters(L, g):
    out = []
    for i in range(2):
        p = C.c_void_p()
        L.check(L.lib().fdb_group_plan(g, i, C.byref(p)))
        out.append(counters(L, p))
    return out


def group_fn(L, g, t):
    p = C.c_void_p()
    L.check(L.lib().fdb_group_plan(g, 0, C.byref(p)))
    return fn_for(L, p, t)


def group_accepted(L, name, t, g):
    cls, cx = GROUPS[name][0], 1 if t == "x" else 0
    c = next((c for c in GROUP_TABLE if GROUP_TABLE[c][cls][cx] is None), None)
    if c is None:
        return None
    b = Bufs(L)
    L.check(group_call(L, c, g, group_fn(L, g, t), b))
    return b.result()


@pytest.mark.parametrize("name,t", GROUP_CASES)
@pytest.mark.parametrize("c", list(GROUP_TABLE))
def test_group_call(L, c, name, t):
    want = GROUP_TABLE[c][GROUPS[name][0]][1 if t == "x" else 0]
    g = make_group(L, name, t)
    try:
        f = group_fn(L, g, t)
        before = group_counters(L, g)
        st = group_call(L, c, g, f, Bufs(L))
        torch.cuda.synchronize()
        msg = L.lib().fdb_last_error().decode()
        if want is None:
            assert st == L.FDB_OK, f"{c} on {name}/{t}: refused with {st}: {msg}"
            return
        assert (st, msg) == (getattr(L, f"FDB_ERR_{want[0]}"), want[1])
        assert f.calls == 0 and group_counters(L, g) == before
        got = group_accepted(L, name, t, g)
    finally:
        L.lib().fdb_group_destroy(g)
    if got is not None:
        g = make_group(L, name, t)
        try:
            assert np.array_equal(got, group_accepted(L, name, t, g))
        finally:
            L.lib().fdb_group_destroy(g)
