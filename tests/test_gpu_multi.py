"""Multi-GPU parity (needs >= 2 GPUs: run under `gpurun --gpus 2`; skipped on a single-GPU box).
One process per GPU (NCCL); colours sharded over the ranks; both exchange modes; every rank must end with the
complete Jacobian, bit-identical to the single-process CPU oracle fed the device-computed step sizes."""
import ctypes as C
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _ell_problem(n, K, Cc, seed):
    rng = np.random.default_rng(seed)
    per = n // Cc
    colors = np.argsort(rng.random((n, Cc)), axis=1)[:, :K]
    which = rng.integers(0, per, size=(n, K))
    cols = (which * Cc + colors).astype(np.int32)
    coef = rng.uniform(-1, 1, size=(n, K))
    return cols, coef


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import scipy.sparse as sps
        import _bootstrap
        pkg = _bootstrap.load_package()
        from _util import assert_same_bits
        from finitediff_jl_b200 import distributed as fdist
        from oracle import fd_oracle as orc
        L = pkg._lib
        n, K, Cc = 64 * 300, 8, 64
        cols, coef = _ell_problem(n, K, Cc, 11)
        A = sps.csc_matrix((np.ones(n * K), (np.repeat(np.arange(n), K), cols.reshape(-1))), shape=(n, n))
        A.sort_indices()
        colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
        cv = (np.arange(n, dtype=np.int64) % Cc) + 1
        xh = orc.fill_x(n, 77)
        colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)   # ELL layout [K][m]
        d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
        octx = orc.SynthEllCtx(n, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
        for fdtype in ("forward", "central"):
            for mode in ("p2p", "nccl"):
                for partition, gather in ((0, "all"), (1, "all"), (0, "root"), (1, "all_p2p")):
                    if gather != "all" and mode != "p2p":
                        continue
                    x = torch.from_numpy(xh).to(dev)
                    J = pkg.SparseMatrixCSC(n, n, torch.from_numpy(colptr), torch.from_numpy(rowval),
                                            torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
                    ctx = L.EllCtx(n, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
                    f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx)
                    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J, rank=rank, world=world, partition=partition)
                    sh = fdist.ShardedJacobian(J, cache, n, dev, mode=mode, gather=gather,
                                               barrier="nccl" if (partition == 1 and gather == "all") else "device")
                    assert sh.mode == mode, getattr(sh, "_fallback_reason", "")
                    for _ in range(2):
                        sh.run(f, x)
                    torch.cuda.synchronize()
                    plan = cache._last_plan
                    info = plan.info()
                    ec = fdist.entry_colors_csc(colptr, cv)
                    counts = np.bincount(ec, minlength=Cc)
                    assert np.array_equal(plan.color_owner(), fdist.partition_colors(Cc, world, counts, partition))
                    assert info["n_local_colors"] == int((plan.color_owner() == rank).sum())
                    eps = plan.eps()
                    ref = np.full(A.nnz, np.nan)
                    orc.jacobian(orc.Problem.csc_same(n, n, colptr, rowval), ref, orc.native_fn("synth_ellrows"), xh.copy(),
                                 fdtype=0 if fdtype == "forward" else 1, colorvec=cv, eps_override=eps, ctx=octx)
                    got = J.nzval.cpu().numpy()
                    if gather != "root" or rank == 0:
                        assert_same_bits(got, ref, f"rank {rank} {fdtype} {mode} partition={partition} {gather}", allow_nan=False)
                    else:   # gather="root": a non-root rank stores straight into rank 0's nzval; its own buffer is untouched
                        assert np.isnan(got).all()
                    per_call = ctx.calls // 2
                    assert per_call == (info["n_local_colors"] + 1 if fdtype == "forward" else 2 * info["n_local_colors"])
                    sh.close()
        # dense column-sharded plan: each rank computes its column slab
        nd = 257
        w = np.random.default_rng(2).random(nd)
        d_w = torch.from_numpy(w).to(dev)
        bs = torch.zeros(8, dtype=torch.float64, device=dev)
        xd = orc.fill_x(nd, 5)
        x = torch.from_numpy(xd).to(dev)
        ctx = L.Rank1Ctx(nd, d_w.data_ptr(), bs.data_ptr(), 4, 0)
        o = L.PlanOpts(fdtype=1, device=rank, max_batch=4, rank=rank, world=world)
        h = C.c_void_p()
        L.check(L.lib().fdb_plan_create_dense(C.byref(h), nd, nd, nd, C.byref(o)))
        plan = pkg.Plan(h.value)
        b, e = plan.dense_range()
        Jslab = torch.full((nd * (e - b),), float("nan"), dtype=torch.float64, device=dev)
        L.check(L.lib().fdb_jacobian(plan.handle, C.cast(L.synth().fdbs_rank1, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p),
                                     x.data_ptr(), Jslab.data_ptr(), None, None, float("nan"), float("nan"), 1.0, None))
        torch.cuda.synchronize()
        ref = np.zeros(nd * nd)
        orc.jacobian(orc.Problem.dense(nd, nd), ref, orc.native_fn("synth_rank1"), xd.copy(), fdtype=1,
                     ctx=orc.SynthRank1Ctx(nd, w.ctypes.data_as(C.POINTER(C.c_double)), 1))
        assert_same_bits(Jslab.cpu().numpy(), ref[b * nd: e * nd], f"rank {rank} dense slab", allow_nan=False)
        assert ctx.calls == 2 * (e - b)
        # column-block shards (few-colour problem): every rank owns a block of columns; J sharded, then gathered on rank 0
        from _util import cyc_colors, tridiag_csc
        nt = 30011
        cpt, rvt = tridiag_csc(nt)
        cvt = cyc_colors(nt, 3)
        xt = torch.from_numpy(orc.fill_x(nt, 9)).to(dev)
        for fdtype in ("forward", "central"):
            octx_t = orc.SynthTridiagCtx(nt, 1)
            for gather in (None, "root"):
                Jt = pkg.SparseMatrixCSC(nt, nt, torch.from_numpy(cpt).to(dev), torch.from_numpy(rvt).to(dev),
                                         torch.full((len(rvt),), float("nan"), dtype=torch.float64, device=dev))
                keep = []

                def factory(r0, r1, x0, x1):
                    c = L.TridiagRowsCtx(nt, r0, r1 - r0, x0, 0)
                    keep.append(c)
                    return pkg.NativeFn(C.cast(L.synth().fdbs_tridiag_rows, C.c_void_p).value, c)

                cs = fdist.ColumnShardedJacobian(Jt, cvt, fdtype, dev, factory, gather=gather)
                for _ in range(2):
                    cs.run(xt)
                torch.cuda.synchronize()
                dist.barrier()
                eps = cs.eps_plan.plan.eps()
                ref = np.full(len(rvt), np.nan)
                orc.jacobian(orc.Problem.csc_same(nt, nt, cpt, rvt), ref, orc.native_fn("synth_tridiag"), orc.fill_x(nt, 9),
                             fdtype=0 if fdtype == "forward" else 1, colorvec=cvt, eps_override=eps, ctx=octx_t)
                got = Jt.nzval.cpu().numpy()
                if gather == "root" and rank == 0:
                    assert_same_bits(got, ref, f"column shards gathered on root, {fdtype}", allow_nan=False)
                elif gather is None:
                    b = cs.block
                    assert_same_bits(got[b.p0:b.p1], ref[b.p0:b.p1], f"rank {rank} column block {fdtype}", allow_nan=False)
                    assert np.isnan(got[:b.p0]).all() and np.isnan(got[b.p1:]).all()
                cs.close()
        (Path(out_dir) / f"ok_{rank}").write_text("ok")
    finally:
        dist.destroy_process_group()


def test_two_gpu_sharded_colors(tmp_path, oracle):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok_{r}").exists() for r in range(world))
