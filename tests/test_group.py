"""The multi-GPU code path on ANY box (run with -m gpu; a single GPU is enough).

fdb_group_* drives n plans (rank i of n) from one process; device ordinals may repeat, so devices = [0, 0] exercises on
one GPU exactly what N GPUs run: colour ownership, the non-FULL scatter variants, the colour-major entry lists, the
zero bucket of rank 0, stores into ONE shared Jacobian buffer, dense column blocks, the event ordering — bit-compared
with the CPU oracle (fed the device-computed step sizes) and with the single-plan GPU result.  With >= 2 GPUs the same
tests also run over [0, 1] (peer access over NVLink).  fdb_sync (the device-side barrier used one-process-per-GPU) is
exercised with two ranks living in one process on two streams.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, cyc_colors, tridiag_csc  # noqa: E402

FD = {"forward": 0, "central": 1}


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
    sets = [[0, 0], [0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets += [[0, 1], [1, 0, 1]]
    return sets


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))


def ell_problem(n, K, Cc, seed):
    rng = np.random.default_rng(seed)
    per = n // Cc
    colors = np.argsort(rng.random((n, Cc)), axis=1)[:, :K]
    which = rng.integers(0, per, size=(n, K))
    cols = (which * Cc + colors).astype(np.int32)
    coef = rng.uniform(-1, 1, size=(n, K))
    return cols, coef


def ell_setup(pkg, oracle, n, K, Cc, devices):
    import scipy.sparse as sps
    cols, coef = ell_problem(n, K, Cc, 11)
    A = sps.csc_matrix((np.ones(n * K), (np.repeat(np.arange(n), K), cols.reshape(-1))), shape=(n, n))
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)
    per_dev = {}
    for d in set(devices):
        dev = torch.device("cuda", d)
        per_dev[d] = (torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev))
    octx = oracle.SynthEllCtx(n, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    return A, colptr, rowval, per_dev, octx, (colsT, coefT)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("partition", [0, 1])
@pytest.mark.parametrize("strategy", [0, 1])
def test_group_csc_colour_shards(pkg, fdist, oracle, fdtype, partition, strategy):
    """C4 shape (random sparse, 64 colours) sharded over group members; strategy 0 = auto (colour-major lists when
    sharded), 1 = the fused storage-order pass with ownership tests (FULL = false)."""
    L = pkg._lib
    n, K, Cc = 64 * 300, 8, 64
    for devices in device_sets():
        A, colptr, rowval, per_dev, octx, keep = ell_setup(pkg, oracle, n, K, Cc, devices)
        cv = cyc_colors(n, Cc)
        cv[5::97] = 0                        # a few columns without a valid colour: rank 0's zero bucket
        root = torch.device("cuda", devices[0])
        xh = oracle.fill_x(n, 77)
        x = torch.from_numpy(xh).to(root)
        J = pkg.SparseMatrixCSC(n, n, t64(colptr), t64(rowval), torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=root))
        ctxs = [L.EllCtx(n, K, per_dev[d][0].data_ptr(), per_dev[d][1].data_ptr(), 0) for d in devices]
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, c) for c in ctxs]
        g = fdist.GroupJacobian(J, cv, fdtype, devices, partition=partition, strategy=strategy)
        for _ in range(2):
            J.nzval.fill_(float("nan"))
            g.run(fs, x)
            g.synchronize()
        eps = g.plans[0].eps()
        ref = np.full(A.nnz, np.nan)
        r = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows"), xh.copy(),
                            fdtype=FD[fdtype], colorvec=cv, eps_override=eps, ctx=octx)
        got = J.nzval.cpu().numpy()
        assert_same_bits(got, ref, f"devices={devices} {fdtype} partition={partition} strategy={strategy}", allow_nan=False)
        # ownership is a partition of the colours; every member evaluated exactly its share (+ f(x) in forward mode)
        owner = g.plans[0].color_owner()
        ec = fdist.entry_colors_csc(colptr, cv)
        counts = np.bincount(ec[ec >= 0], minlength=Cc)
        assert np.array_equal(owner, fdist.partition_colors(Cc, len(devices), counts, partition))
        total = 0
        for i, c in enumerate(ctxs):
            nl = g.plans[i].info()["n_local_colors"]
            assert nl == int((owner == i).sum())
            assert c.calls // 2 == (nl + 1 if fdtype == "forward" else 2 * nl)
            total += nl
            assert_same_bits(g.plans[i].eps(), eps, allow_nan=False)               # every member derives the same step sizes
            assert g.plans[i].info()["strategy"] == (1 if strategy == 0 else 0)
        assert total == Cc and r["fcalls"] == (Cc + 1 if fdtype == "forward" else 2 * Cc)
        g.close()


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_group_matches_single_plan_and_graph(pkg, fdist, oracle, fdtype):
    """sharded == unsharded, bit for bit (the drift replay is closed-form), with CUDA-graph replay per member"""
    L = pkg._lib
    N = 20011
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 7)
    for devices in device_sets():
        root = torch.device("cuda", devices[0])
        xh = oracle.fill_x(N, 3)
        x = torch.from_numpy(xh).to(root)
        J1 = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=root))
        c1 = L.TridiagCtx(N, 0)
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J1)
        with torch.cuda.device(root):
            pkg.finite_difference_jacobian_(J1, pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, c1), x, cache)
        J2 = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=root))
        ctxs = [L.TridiagCtx(N, 0) for _ in devices]
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, c) for c in ctxs]
        g = fdist.GroupJacobian(J2, cv, fdtype, devices, use_graph=True)
        for _ in range(3):
            J2.nzval.fill_(float("nan"))
            g.run(fs, x)
            g.synchronize()
        assert_same_bits(J1.nzval, J2.nzval, f"devices={devices}", allow_nan=False)
        g.close()


def lap5_colors(g):
    return np.array([((i) + 2 * (j)) % 5 + 1 for j in range(g) for i in range(g)], dtype=np.int64)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_group_banded(pkg, fdist, oracle, fdtype):
    """BandedMatrix sparsity (whole-band fill) sharded by colour: band-data target and dense-J target (the root
    zero-fills the shared dense J once, members only store)."""
    L = pkg._lib
    for gsz, devices in [(64, [0, 0]), (65, [0, 0, 0])] + ([(64, [0, 1])] if torch.cuda.device_count() >= 2 else []):
        n = gsz * gsz
        cv = lap5_colors(gsz)
        root = torch.device("cuda", devices[0])
        xh = oracle.fill_x(n, 0x5EED + 3)
        x = torch.from_numpy(xh).to(root)
        ctxs = [L.Lap5Ctx(gsz, 0) for _ in devices]
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_lap5, C.c_void_p).value, c) for c in ctxs]
        Jb = pkg.BandedMatrix(n, n, gsz, gsz, device=root)
        Jb.data.fill_(float("nan"))
        g = fdist.GroupJacobian(Jb, cv, fdtype, devices)
        g.run(fs, x)
        g.synchronize()
        refb = np.full((2 * gsz + 1) * n, np.nan)
        oracle.jacobian(oracle.Problem.banded(n, n, gsz, gsz), refb, oracle.native_fn("synth_lap5"), xh.copy(),
                        fdtype=FD[fdtype], colorvec=cv, eps_override=g.plans[0].eps(), ctx=oracle.SynthLap5Ctx(gsz, 1))
        assert_same_bits(Jb.data.cpu().numpy(), refb, f"band data, devices={devices}", allow_nan=False)
        g.close()
        Jd = pkg.zeros_colmajor(n, n, root)
        Jd.fill_(float("nan"))
        g = fdist.GroupJacobian(Jd, cv, fdtype, devices, sparsity=pkg.BandedMatrix(n, n, gsz, gsz, data=torch.zeros(1), device=root))
        g.run(fs, x)
        g.synchronize()
        refd = np.zeros(n * n)
        oracle.jacobian(oracle.Problem.banded_to_dense(n, n, gsz, gsz), refd, oracle.native_fn("synth_lap5"), xh.copy(),
                        fdtype=FD[fdtype], colorvec=cv, eps_override=g.plans[0].eps(), ctx=oracle.SynthLap5Ctx(gsz, 1))
        assert_same_bits(Jd.cpu().numpy().reshape(-1, order="F"), refd, f"dense target, devices={devices}", allow_nan=False)
        g.close()


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_group_dense_column_blocks(pkg, fdist, oracle, fdtype):
    """sparsity === nothing: contiguous column blocks per member (BASELINE config 5's partition), batched f!"""
    L = pkg._lib
    n = 515
    w = np.random.default_rng(2).random(n)
    for devices in device_sets():
        root = torch.device("cuda", devices[0])
        batch = 8
        keep, ctxs = [], []
        for d in devices:
            dev = torch.device("cuda", d)
            d_w = torch.from_numpy(w).to(dev)
            bs = torch.zeros(((n + 1023) // 1024) * batch, dtype=torch.float64, device=dev)
            keep.append((d_w, bs))
            ctxs.append(L.Rank1Ctx(n, d_w.data_ptr(), bs.data_ptr(), batch, 0))
        fs = [pkg.NativeFn(C.cast(L.synth().fdbs_rank1, C.c_void_p).value, c, max_batch=batch) for c in ctxs]
        xh = oracle.fill_x(n, 0x5EED + 5)
        x = torch.from_numpy(xh).to(root)
        J = pkg.zeros_colmajor(n, n, root)
        J.fill_(float("nan"))
        g = fdist.GroupJacobian(J, None, fdtype, devices, max_batch=batch)
        g.run(fs, x)
        g.synchronize()
        ref = np.zeros(n * n)
        r = oracle.jacobian(oracle.Problem.dense(n, n), ref, oracle.native_fn("synth_rank1"), xh.copy(), fdtype=FD[fdtype],
                            ctx=oracle.SynthRank1Ctx(n, w.ctypes.data_as(C.POINTER(C.c_double)), 1))
        assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, f"devices={devices}", allow_nan=False)
        cols = 0
        for i, c in enumerate(ctxs):
            b, e = g.plans[i].dense_range()
            cols += e - b
            assert c.calls == (e - b) * (1 if fdtype == "forward" else 2) + (1 if fdtype == "forward" else 0)
        assert cols == n and r["fcalls"] == (n + 1 if fdtype == "forward" else 2 * n)
        g.close()


def test_group_python_callables(pkg, fdist, oracle):
    """Python f!(fx, x) per member (tensors arrive on that member's device)"""
    N = 301
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    devices = [0, 0]
    root = torch.device("cuda", 0)
    xh = oracle.fill_x(N, 4)
    x = torch.from_numpy(xh).to(root)
    calls = [0, 0]

    def make(i):
        def f(fx, xx):
            calls[i] += 1
            fx[1:-1] = (xx[:-2] - 2 * xx[1:-1]) + xx[2:]
            fx[0] = -2 * xx[0] + xx[1]
            fx[-1] = xx[-2] - 2 * xx[-1]
        return f

    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=root))
    g = fdist.GroupJacobian(J, cv, "forward", devices)
    g.run([make(0), make(1)], x)
    g.synchronize()
    assert calls == [3, 2]                                   # colours {1,3} + f(x) on member 0, colour {2} + f(x) on member 1
    dense = J.to_dense()
    exact = np.diag(-2 * np.ones(N)) + np.diag(np.ones(N - 1), 1) + np.diag(np.ones(N - 1), -1)
    assert np.max(np.abs(dense - exact)) < 1e-6
    g.close()


_BARRIER_SCRIPT = r"""
import ctypes as C, sys
sys.path.insert(0, {root!r})
import torch, _bootstrap
pkg = _bootstrap.load_package()
L = pkg._lib
lib = L.lib()
dev = torch.device("cuda:0")
hs, flags = [], []
for r in range(2):
    h = C.c_void_p()
    L.check(lib.fdb_sync_create(C.byref(h), r, 2, 0))
    p = C.c_void_p()
    L.check(lib.fdb_sync_flags(h, C.byref(p)))
    hs.append(h)
    flags.append(p.value)
for r in range(2):
    arr = (C.c_void_p * 2)(flags[0], flags[1])
    L.check(lib.fdb_sync_set_peers(hs[r], arr))
s0, s1 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
payload = torch.zeros(2, dtype=torch.float64, device=dev)
seen = torch.zeros(2, dtype=torch.float64, device=dev)
# load every kernel the loop launches BEFORE a barrier kernel can be spinning: with CUDA's lazy module loading the first
# launch of a kernel synchronises the context, which would wait for the spinning kernel, which waits for the launch
for st in (s0, s1):
    with torch.cuda.stream(st):
        payload[0:1].fill_(0.0)
        seen[0:1].copy_(payload[1:2])
torch.cuda.synchronize()
for it in range(1, 6):
    with torch.cuda.stream(s0):
        payload[0:1].fill_(float(it))
        L.check(lib.fdb_sync_barrier(hs[0], C.c_void_p(s0.cuda_stream)))
        seen[0:1].copy_(payload[1:2])           # rank 0 reads what rank 1 wrote before ITS barrier
        L.check(lib.fdb_sync_barrier(hs[0], C.c_void_p(s0.cuda_stream)))
    with torch.cuda.stream(s1):
        payload[1:2].fill_(float(10 * it))
        L.check(lib.fdb_sync_barrier(hs[1], C.c_void_p(s1.cuda_stream)))
        seen[1:2].copy_(payload[0:1])
        L.check(lib.fdb_sync_barrier(hs[1], C.c_void_p(s1.cuda_stream)))
    torch.cuda.synchronize()
    assert seen.tolist() == [10.0 * it, float(it)], seen.tolist()
for h in hs:
    L.check(lib.fdb_sync_destroy(h))
print("barrier-ok")
"""


def test_device_barrier_two_ranks_one_process(pkg):
    """fdb_sync: two ranks in one process on two streams — each barrier kernel signals the other rank's flag block and
    waits for its own; ordering is checked through a payload written before the barrier.  Run in a fresh process with
    CUDA_DEVICE_MAX_CONNECTIONS=32: a barrier kernel SPINS until its peer has signalled, so the two streams must not share
    a hardware work queue, and every kernel is loaded up front (lazy module loading synchronises the context).  In a real
    job the ranks are separate processes / GPUs and cannot queue behind each other."""
    import os
    import subprocess
    import sys
    from pathlib import Path
    root = str(Path(__file__).resolve().parent.parent)
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32", CUDA_MODULE_LOADING="EAGER")
    r = subprocess.run([sys.executable, "-c", _BARRIER_SCRIPT.format(root=root)], env=env, capture_output=True, text=True, timeout=240)
    assert r.returncode == 0 and "barrier-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
