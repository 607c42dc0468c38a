"""N>1 path on CPU: world_size-2 gloo run of the colour-partition + owned-entry exchange logic
(finitediff.jl_b200/distributed.py), with the CPU oracle standing in for each rank's device compute.
The same partition_colors / GatherPlan / allgather_owned code runs on the GPUs in "nccl" mode; the "p2p" mode and the
plan-side partition are covered by tests/test_gpu_multi.py on real GPUs."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, mode, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import _bootstrap
        pkg = _bootstrap.load_package()
        from finitediff_jl_b200 import distributed as fdist
        from oracle import fd_oracle as orc
        from _util import assert_same_bits, tridiag_csc, cyc_colors, f_tridiag
        N, C_ = 600, 7
        colptr, rowval = tridiag_csc(N)
        cv = cyc_colors(N, C_)
        cv[5] = 0                                          # a column without a valid colour: its entries stay 0
        x = orc.fill_x(N, 123)
        full = np.full(len(rowval), np.nan)
        orc.jacobian(orc.Problem.csc_same(N, N, colptr, rowval), full, f_tridiag, x.copy(), colorvec=cv)
        ec = fdist.entry_colors_csc(colptr, cv)
        counts = np.bincount(ec[ec >= 0], minlength=C_)
        owner = fdist.partition_colors(C_, world, counts, mode)
        # every colour has exactly one owner; LPT balances the entry counts
        assert owner.min() >= 0 and owner.max() < world
        gp = fdist.GatherPlan(ec, owner, world, "cpu")
        assert sum(int(i.numel()) for i in gp.idx) == len(rowval)
        # this rank "computes" only the entries of its colours (plus the invalid-colour zeros on rank 0)
        mine = torch.full((len(rowval),), float("nan"), dtype=torch.float64)
        sel = gp.idx[rank]
        mine[sel] = torch.from_numpy(full)[sel]
        fdist.allgather_owned(mine, gp, rank)
        got = mine.numpy()
        assert_same_bits(got, full, f"rank {rank}: gathered Jacobian differs", allow_nan=False)
        loads = [int(counts[owner == r].sum()) for r in range(world)]
        (Path(out_dir) / f"ok_{rank}").write_text(f"{loads}")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", [0, 1])
def test_two_rank_gloo_color_partition_and_gather(tmp_path, mode, oracle):
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, mode, str(tmp_path)), nprocs=world, join=True)
    assert (tmp_path / "ok_0").exists() and (tmp_path / "ok_1").exists()
    loads = eval((tmp_path / "ok_0").read_text())
    if mode == 1:
        assert abs(loads[0] - loads[1]) <= max(loads) * 0.35


def test_partition_rules():
    import _bootstrap
    _bootstrap.load_package()
    from finitediff_jl_b200 import distributed as fdist
    assert fdist.partition_colors(5, 1).tolist() == [0] * 5
    assert fdist.partition_colors(7, 3).tolist() == [0, 1, 2, 0, 1, 2, 0]
    own = fdist.partition_colors(6, 2, counts=[10, 1, 1, 1, 1, 8], mode=1)
    # LPT: 10 -> r0, 8 -> r1, then the ones alternate onto the lighter rank (ties -> lowest rank)
    assert own[0] == 0 and own[5] == 1
    load = [sum(c for c, o in zip([10, 1, 1, 1, 1, 8], own) if o == r) for r in (0, 1)]
    assert abs(load[0] - load[1]) <= 2
    ec = fdist.entry_colors_csc(np.array([1, 3, 4, 6]), np.array([2, 0, 1]))
    assert ec.tolist() == [1, 1, -1, 0, 0]
