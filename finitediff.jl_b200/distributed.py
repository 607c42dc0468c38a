"""One process per GPU: the colour set of a Jacobian is partitioned over the ranks (SURVEY.md §8e).

Colours are independent units given x (each colour = perturb -> f! -> diff -> scatter into a disjoint set of J slots),
so there is NO collective on the data path until the end, where every rank needs the entries the others computed.
Two implementations of that final exchange:

  "p2p"  (default on NVLink/NVSwitch)  the diff+scatter kernel itself stores every value it owns into rank 0's nzval
         buffer (gather="root": rank 0's buffer is mapped by every rank over CUDA IPC and passed as THE J of plans created
         with shared_j) — compute and gather are one kernel; the ranks are ordered by the C ABI's device-side barrier
         (fdb_sync, DeviceBarrier below), no NCCL call per Jacobian.  gather="all" adds one NCCL broadcast of nzval;
         gather="all_p2p" stores to every peer from the kernel (fine up to 4 GPUs, pathological at 8 — see ShardedJacobian).
  "nccl" (fallback; also what the CPU/gloo tests exercise)  each rank packs the entries it owns into a compact
         buffer, all_gather, then un-permutes into nzval.

torch.distributed is plumbing only (rendezvous, barrier, the fallback all_gather); the hot path is libfdjac_b200.so.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L
from . import api


# ------------------------------------------------------------------------------------------------ host-side partition logic
def partition_colors(n_colors: int, world: int, counts=None, mode: int = 0) -> np.ndarray:
    """Owner rank of every colour — the same deterministic rule as the plan (csrc/fdjac_abi.cu finish_colored_plan):
    mode 0 round-robin; mode 1 LPT (heaviest colour first onto the least-loaded rank, ties -> lowest rank)."""
    owner = np.zeros(n_colors, np.int32)
    if world <= 1:
        return owner
    if mode == 1:
        counts = np.asarray(counts, dtype=np.uint64)
        order = sorted(range(n_colors), key=lambda k: -int(counts[k]))   # stable: ties keep ascending colour
        load = [0] * world
        for k in order:
            best = min(range(world), key=lambda r: (load[r], r))
            owner[k] = best
            load[best] += int(counts[k]) + 1
    else:
        owner[:] = np.arange(n_colors) % world
    return owner


def entry_colors_csc(colptr, colorvec) -> np.ndarray:
    """0-based colour of every CSC entry (colour of its column); -1 where colorvec < 1."""
    colptr = np.asarray(colptr, dtype=np.int64)
    cv = np.asarray(colorvec, dtype=np.int64)
    per_col = np.diff(colptr)
    ec = np.repeat(cv - 1, per_col)
    ec[ec < 0] = -1
    return ec


class GatherPlan:
    """Index lists for the pack / all_gather / unpack exchange of owned Jacobian entries."""

    def __init__(self, entry_color: np.ndarray, owner: np.ndarray, world: int, device):
        self.world = world
        own = np.where(entry_color >= 0, owner[np.clip(entry_color, 0, max(len(owner) - 1, 0))] if len(owner) else 0, 0)
        self.idx: List[torch.Tensor] = []
        for r in range(world):
            self.idx.append(torch.from_numpy(np.nonzero(own == r)[0].astype(np.int64)).to(device))
        self.pad = max((int(i.numel()) for i in self.idx), default=0)

    def pack(self, values: torch.Tensor, rank: int) -> torch.Tensor:
        out = torch.zeros(self.pad, dtype=values.dtype, device=values.device)
        out[: self.idx[rank].numel()] = values.index_select(0, self.idx[rank])
        return out

    def unpack(self, values: torch.Tensor, gathered: List[torch.Tensor], skip_rank: Optional[int] = None):
        for r, g in enumerate(gathered):
            if r == skip_rank:
                continue
            values.index_copy_(0, self.idx[r], g[: self.idx[r].numel()])


def allgather_owned(values: torch.Tensor, gp: GatherPlan, rank: int, group=None):
    """values holds this rank's owned entries in place; on return it holds everybody's (gloo or nccl)."""
    mine = gp.pack(values, rank)
    gathered = [torch.empty_like(mine) for _ in range(gp.world)]
    dist.all_gather(gathered, mine, group=group)
    gp.unpack(values, gathered, skip_rank=rank)
    return values


# ------------------------------------------------------------------------------------------------ device side
class IpcBuffer:
    """A float64 device buffer from a dedicated cudaMalloc (so its CUDA IPC handle maps the buffer itself)."""

    def __init__(self, count: int, device: torch.device):
        self.count = int(count)
        p = C.c_void_p()
        api._call(device, (), L.lib().fdb_device_alloc, C.byref(p), max(self.count, 2) * 8)
        self.ptr = p.value
        self.device = device
        self.tensor = torch.as_tensor(api._DevArray(self.ptr, (self.count,)), device=device)

    def handle(self) -> bytes:
        h = C.create_string_buffer(64)
        L.check(L.lib().fdb_ipc_get_handle(C.c_void_p(self.ptr), h))
        return h.raw

    def free(self):
        if self.ptr:
            with torch.cuda.device(self.device):
                L.lib().fdb_device_free(C.c_void_p(self.ptr))
            self.ptr = 0


class DeviceBarrier:
    """fdb_sync: the device-side barrier that orders one-process-per-GPU ranks without NCCL on the data path — a flag
    block per rank in peer memory (CUDA IPC), one tiny kernel per barrier enqueued on the caller's stream
    (st.release.sys to every peer, ld.acquire.sys until every peer has signalled).  torch.distributed is used once, at
    construction, to exchange the 64-byte IPC handles."""

    def __init__(self, device, group=None):
        self.device = torch.device(device)
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        h = C.c_void_p()
        api._call(self.device, (), L.lib().fdb_sync_create, C.byref(h), self.rank, self.world, api._device_index(self.device))
        self._h = h
        flags = C.c_void_p()
        L.check(L.lib().fdb_sync_flags(self._h, C.byref(flags)))
        mine = C.create_string_buffer(64)
        L.check(L.lib().fdb_ipc_get_handle(flags, mine))
        handles = [None] * self.world
        dist.all_gather_object(handles, mine.raw, group=group)
        self._mapped = []
        ptrs = (C.c_void_p * self.world)()
        with torch.cuda.device(self.device):
            for r, hb in enumerate(handles):
                if r == self.rank:
                    ptrs[r] = flags.value
                    continue
                p = C.c_void_p()
                L.check(L.lib().fdb_ipc_open(hb, C.byref(p)))
                self._mapped.append(p.value)
                ptrs[r] = p.value
            L.check(L.lib().fdb_sync_set_peers(self._h, ptrs))
        dist.barrier(group=group)          # every rank has mapped every flag block before the first signal

    def wait(self, stream=None):
        """Enqueue one barrier on `stream` (default: the current stream of the device)."""
        L.check(L.lib().fdb_sync_barrier(self._h, C.c_void_p(api._stream(stream, self.device))))

    def close(self):
        if self._h is None:
            return
        torch.cuda.synchronize(self.device)
        with torch.cuda.device(self.device):
            for p in self._mapped:
                L.lib().fdb_ipc_close(C.c_void_p(p))
            self._mapped = []
        _barrier(self.group)                     # nobody frees a flag block a peer may still signal
        L.lib().fdb_sync_destroy(self._h)
        self._h = None


def _barrier(group):
    """dist.barrier on `group` at teardown, where the process group may already be gone."""
    try:
        dist.barrier(group=group)
    except Exception:
        pass


class _RootValues:
    """Rank 0's J.nzval mapped into every rank over CUDA IPC.  Rank 0 moves its values into an IpcBuffer (so that the
    handle maps exactly them, and J.nzval is that buffer from then on); every other rank opens rank 0's handle and finds
    the mapping at `ptr` (None on rank 0)."""

    def __init__(self, J: api.SparseMatrixCSC, device, rank: int, world: int, group):
        self.device, self.group = device, group
        self._ipc: Optional[IpcBuffer] = None
        self.ptr = None
        mine = None
        if rank == 0:
            self._ipc = IpcBuffer(J.nzval.numel(), device)
            self._ipc.tensor.copy_(J.nzval)
            J.nzval = self._ipc.tensor
            mine = self._ipc.handle()
        handles = [None] * world
        dist.all_gather_object(handles, mine, group=group)
        if rank != 0:
            p = C.c_void_p()
            api._call(device, (), L.lib().fdb_ipc_open, handles[0], C.byref(p))
            self.ptr = p.value

    def close(self):
        """Unmap, then a barrier, then free: rank 0 frees its buffer only once no rank maps it."""
        if self.ptr:
            with torch.cuda.device(self.device):
                L.lib().fdb_ipc_close(C.c_void_p(self.ptr))
            self.ptr = None
        _barrier(self.group)
        if self._ipc is not None:
            self._ipc.free()
            self._ipc = None


class _Group:
    """What the group classes share: the fdb_group handle, its member plans, one f per member behind one entry point,
    and the joins."""

    def _set_devices(self, devices):
        self.devices = [api._device_index(d) if not isinstance(d, int) else int(d) for d in devices]
        self.root = torch.device("cuda", self.devices[0])

    def _create(self, creator, opts, *args):
        """Adopt the group fdb_group_create_<creator>(&h, n_devices, devices, *args, &opts) creates."""
        devs = (C.c_int * len(self.devices))(*self.devices)
        self._adopt(api._new_handle(f"fdb_group_create_{creator}", len(self.devices), devs, *args, C.byref(opts)))

    def _adopt(self, h):
        lib = L.lib()
        self._h = h
        self._fin = api.weakref.finalize(self, lib.fdb_group_destroy, C.c_void_p(h.value))
        self.plans = []
        for i in range(len(self.devices)):
            p = C.c_void_p()
            L.check(lib.fdb_group_plan(self._h, i, C.byref(p)))
            self.plans.append(api.Plan(p.value, owned=False))
        self._fns = None

    def _member_fns(self, fs, m, n, **kind):
        """(entry address, contexts array, per-member Python wrappers or None) for one f per member.  The ABI takes one f
        and a context per member: NativeFns must share their address; Python callables go through ONE trampoline whose
        context is the member index + 1, forwarding to that member's wrapper (tensors on that member's device)."""
        if len(fs) != len(self.devices):
            raise ValueError("one f! per member")
        if self._fns is None or self._fns[0] is not fs:
            keep = None
            if all(isinstance(f, api.NativeFn) for f in fs):
                wrapped = [api._as_fn(f, m, n, torch.device("cuda", d), 1) for f, d in zip(fs, self.devices)]
            else:
                per = [api._PyFn(f, m, n, torch.device("cuda", d), bool(getattr(f, "batched", False)), **kind)
                       for f, d in zip(fs, self.devices)]

                def tramp(ctx, p_fx, p_x, batch, ldfx, ldx, stream, _per=per):
                    return _per[int(ctx or 1) - 1]._tramp(None, p_fx, p_x, batch, ldfx, ldx, stream)

                keep = L.FDB_FN(tramp)
                wrapped = [(L.fn_address(keep), C.c_void_p(i + 1), per[i]) for i in range(len(per))]
            self._fns = (fs, wrapped, keep)
        wrapped = self._fns[1]
        addr = wrapped[0][0]
        if any(w[0] != addr for w in wrapped):
            raise ValueError("all members must share one f! entry point (contexts may differ per device)")
        ctxs = (C.c_void_p * len(wrapped))(*[C.cast(w[1], C.c_void_p).value if w[1] is not None else None for w in wrapped])
        return addr, ctxs, [w[2] for w in wrapped]

    def synchronize(self):
        for d in set(self.devices):
            torch.cuda.synchronize(d)

    def close(self):
        self.synchronize()
        self._fin()


class GroupJacobian(_Group):
    """ONE process driving several GPUs through fdb_group_* (the C ABI's own multi-GPU entry: no torch.distributed, no
    NCCL): colours (dense: column blocks) are partitioned over `devices`; devices[0] is the root and owns x, J and fx;
    every member's scatter kernel stores the entries it owns straight into the root's J over NVLink.  Device ordinals
    may repeat ([0, 0] runs two members on one GPU — the same code path on a single-GPU box).

    fs: one f! per member (NativeFn whose context lives on that member's device, or a Python callable)."""

    def __init__(self, J, colorvec, fdtype, devices, *, sparsity=api._DEFAULT, **plan_kw):
        self._set_devices(devices)
        self.J, self.fdtype = J, fdtype
        if sparsity is api._DEFAULT:
            sparsity = J if api._has_sparsestruct(J) else None
        kind, args, self._keep = api._plan_route(J, sparsity, colorvec)
        if kind == "coo":
            raise TypeError(f"GroupJacobian: unsupported sparsity type {type(sparsity)}")
        if kind == "dense_colorvec":
            kind, args = "dense", args[:3]          # a dense group splits the columns 1:n; colorvec is not read
        self._create(kind, api._opts(api._fdtype_code(fdtype), self.devices[0], **plan_kw), *args)

    def run(self, fs, x, fx=None, f_in=None, *, relstep=None, absstep=None, dir=True, stream=None):
        m, n = api._shape_of(self.J)
        addr, ctxs, pyfns = self._member_fns(fs, m, n)
        api._call(self.root, pyfns, L.lib().fdb_group_jacobian, self._h, addr, ctxs, x.data_ptr(),
                  api._j_values(self.J).data_ptr(), None if fx is None else fx.data_ptr(),
                  None if f_in is None else f_in.data_ptr(), *api._steps(relstep, absstep), float(dir),
                  C.c_void_p(api._stream(stream, self.root)))


class GroupHessian(_Group):
    """finite_difference_hessian! on several GPUs from ONE process (fdb_group_create_hessian / fdb_group_hessian): the
    i-blocks of the reference's point sequence are split over `devices` in contiguous, point-balanced ranges (member i's
    is plans[i].dense_range()); devices[0] is the root and owns x, H and fx; every non-empty member evaluates f(x) and
    its own points and stores the entries it owns straight into the root's H.  H is bit-identical to one device.  Device
    ordinals may repeat ([0, 0] runs two members on one GPU).

    plan_kw: max_batch, scratch_bytes, use_graph (per member), fdtype (only "hcentral" is built)."""

    def __init__(self, n, devices, *, ldH=None, fdtype="hcentral", **plan_kw):
        self._set_devices(devices)
        self.n = int(n)
        self.ldH = max(self.n, 1) if ldH is None else int(ldH)
        self._create("hessian", api._opts(api._hessian_fdtype_code(fdtype), self.devices[0], **plan_kw), self.n, self.ldH)

    def run(self, fs, x, H, fx=None, *, relstep=None, absstep=None, stream=None):
        """fs: one f per member — a NativeFn (batched fdb_fn with m = 1, context on that member's device) or a Python
        f(x) -> scalar on that member's device (f.batched = True: (batch, n) in, (batch,) out).  x, H (column-major n x n,
        leading dimension ldH) and fx (optional 1-element tensor receiving f(x)) live on devices[0]."""
        xv = api._scalar_x(x)
        if xv.numel() != self.n or xv.device != self.root:
            raise ValueError(f"x must hold {self.n} values on {self.root}")
        ld = api._colmajor_square(H, self.n)
        if (self.n > 1 and ld != self.ldH) or H.device != self.root:      # n <= 1: one element, any leading dimension
            raise ValueError(f"H must be column-major with leading dimension {self.ldH} on {self.root}")
        if fx is not None and (not api._is_cuda(fx) or fx.dtype != torch.float64 or fx.numel() != 1):
            raise TypeError("fx must be a 1-element float64 CUDA tensor")
        addr, ctxs, pyfns = self._member_fns(fs, 1, self.n, scalar=True)
        api._call(self.root, pyfns, L.lib().fdb_group_hessian, self._h, addr, ctxs, xv.data_ptr(),
                  H.data_ptr() if self.n > 0 else None, None if fx is None else fx.data_ptr(),
                  *api._steps(relstep, absstep), C.c_void_p(api._stream(stream, self.root)))


def dense_column_blocks(n: int, world: int) -> List[tuple]:
    """[(col_begin, col_end)] of every member of a dense group (csrc/fdjac_abi.cu create_dense): member r owns the
    contiguous columns [min(n, r*p), min(n, (r+1)*p)) with p = ceil(n / world).  Every column costs the same f calls, so
    the largest block, ceil(n / world) columns, is as small as any split makes it; trailing members may be empty."""
    if n < 0 or world < 1:
        raise ValueError("n must be >= 0 and world >= 1")
    p = -(-n // world)
    return [(min(n, r * p), min(n, (r + 1) * p)) for r in range(world)]


class GroupGradient(_Group):
    """finite_difference_gradient!(df, f, x, cache) for a vector x on several GPUs from ONE process: the dense group with
    m = 1 and ldJ = 1 (fdb_group_create_dense / fdb_group_jacobian), df as J.  Member i owns the contiguous components
    plans[i].dense_range() (dense_column_blocks) and writes exactly those entries of the root's df; devices[0] is the
    root and owns x and df.  df is bit-identical to finite_difference_gradient_ on one device.  Device ordinals may repeat
    ([0, 0] runs two members on one GPU).

    fdtype: "forward" or "central" ("complex" builds, and its run raises FdbError(FDB_ERR_UNSUPPORTED) before any f
    call).  plan_kw: max_batch, scratch_bytes, use_graph (per member)."""

    def __init__(self, n, devices, fdtype="central", **plan_kw):
        if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 0:
            raise ValueError("n must be a non-negative integer")
        if len(devices) < 1:
            raise ValueError("a group needs at least one device")
        self.n = int(n)
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        self._code = api._fdtype_code(self.fdtype)
        self._set_devices(devices)
        self._create("dense", api._opts(self._code, self.devices[0], **plan_kw), 1, self.n, 1)
        self.columns = dense_column_blocks(self.n, len(self.devices))      # member i: plans[i].dense_range()

    def run(self, fs, x, df, fx=None, *, relstep=None, absstep=None, dir=True, stream=None):
        """fs: one f per member — a NativeFn (batched fdb_fn with m = 1, context on that member's device) or a Python
        f(x) -> scalar on that member's device (f.batched = True: (batch, n) in, (batch,) out).  x and df: float64 CUDA
        vectors of length n on devices[0]; x is never modified.  Forward mode: f(x) is evaluated once, by fs[0] at the
        root, unless fx (a number, or a 1-element float64 CUDA tensor on devices[0]) is given (gradients.jl:409-410); it
        is passed to every member as f_in, so a call makes 1 + n evaluations (n with fx).  fx is not read otherwise."""
        if len(fs) != len(self.devices):
            raise ValueError("one f per member")
        xv = api._scalar_x(x)
        dv = api._scalar_x(df, "df")
        if xv.numel() != self.n or xv.device != self.root:
            raise ValueError(f"x must hold {self.n} values on {self.root}")
        if dv.numel() != self.n or dv.device != self.root:
            raise ValueError(f"df must hold {self.n} values on {self.root}")
        if df.reshape(-1).data_ptr() != dv.data_ptr():
            raise ValueError("df must be contiguous")
        if isinstance(fx, torch.Tensor):
            if not api._is_cuda(fx) or fx.dtype != torch.float64 or fx.numel() != 1 or fx.device != self.root:
                raise TypeError(f"fx must be a number or a 1-element float64 CUDA tensor on {self.root}")
        elif fx is not None and not api._is_number(fx):
            raise TypeError("fx must be a number or a 1-element float64 CUDA tensor")
        addr, ctxs, pyfns = self._member_fns(fs, 1, self.n, scalar=True)
        stream = api._stream(stream, self.root)
        fin = None
        if self._code == L.FDB_FORWARD:
            # a number (or nothing: f(x) below) goes into the root's one device slot, a stable pointer for graphs
            fin = fx if isinstance(fx, torch.Tensor) else api._device_slot(self, "_fx_slot", self.root, stream, fx)
            if fx is None:
                with torch.cuda.device(self.root):
                    self._root_fx(fs[0], pyfns[0], xv, fin, stream)
        api._call(self.root, pyfns, L.lib().fdb_group_jacobian, self._h, addr, ctxs, xv.data_ptr() or None,
                  dv.data_ptr() or None, None, None if fin is None else fin.data_ptr(), *api._steps(relstep, absstep),
                  float(dir), C.c_void_p(stream))

    @staticmethod
    def _root_fx(f0, py, xv, fin, stream):
        """f(x) by member 0's f, into fin on the root's stream (fx0 = f(x), gradients.jl:410)"""
        if py is None:
            api._native_call(f0, fin, xv, stream)
            return
        if py._tramp(None, fin.data_ptr(), xv.data_ptr() or None, 1, 1, max(xv.numel(), 1), stream) != 0:
            exc, py.exc = py.exc, None
            raise exc


class GroupJacobianOOP(_Group):
    """The out-of-place finite_difference_jacobian(f, x, cache, f_in; ...) on several GPUs from ONE process
    (fdb_group_create_oop_* / fdb_group_jacobian_oop): the colours (dense branch: column blocks of the maximum(colorvec)
    quotient columns) are split over `devices` as GroupJacobian splits them; devices[0] is the root and owns x and the
    result.  Every member writes exactly its own slots of the root's result; a sparse result is compacted by the root once
    every member has finished.  The result is bit-identical to finite_difference_jacobian on one device.  Device ordinals
    may repeat ([0, 0] runs two members on one GPU).

    fdtype, colorvec, sparsity, jac_prototype: as finite_difference_jacobian takes them (colorvec None: 1:length(x)).
    The member plans are built on the first run for the (rows, length(x)) it sees, and rebuilt when those change.
    plan_kw: max_batch, scratch_bytes, partition, use_graph (per member)."""

    def __init__(self, devices, fdtype="forward", colorvec=None, sparsity=None, jac_prototype=None, **plan_kw):
        self._set_devices(devices)
        self.fdtype, self.colorvec, self.sparsity, self.jac_prototype = fdtype, colorvec, sparsity, jac_prototype
        self.kind, self.pm, self.pn = api._oop_kind(sparsity, jac_prototype)
        self.csr = api._oop_csr(sparsity, jac_prototype)
        self._code = api._fdtype_code(fdtype)
        self._plan_kw = plan_kw
        self._key = None

    def _build(self, m, n):
        if self._key == (m, n):
            return
        if self._key is not None:
            self.close()
        o = api._opts(self._code, self.devices[0], **self._plan_kw)
        suffix, args, self._keep = api._oop_plan_route(self.kind, self.sparsity, self.colorvec, self.pn, m, n,
                                                            self.csr)
        with torch.cuda.device(self.root):
            self._create(f"oop_{suffix}", o, *args)
        self._key = (m, n)

    def run(self, fs, x, f_in=None, *, relstep=None, absstep=None, dir=True, stream=None):
        """fs: one f per member — an out-of-place Python f(x) -> CUDA tensor (f.batched = True: (batch, n) -> (batch, m))
        on that member's device, or a NativeFn (the in-place fdb_fn, context on that member's device).  x (float64, on
        devices[0]) is never modified.  In forward mode without f_in, f(x) is evaluated once, by fs[0] at the root, and
        passed on as f_in (jacobians.jl:299-300), so the members evaluate only their colours.  Rows of the result: those
        of the sparsity or prototype, else of f_in or f(x), else length(x).  Returns what finite_difference_jacobian
        returns: a dense column-major tensor, or a SparseMatrixCSC (SparseMatrixCSR with a CSR prototype) sized to the kept
        entries (one host sync)."""
        if not api._is_cuda(x) or x.dtype != torch.float64 or x.device != self.root:
            raise TypeError(f"x must be a float64 CUDA tensor on {self.root}")
        if len(fs) != len(self.devices):
            raise ValueError("one f per member")
        xv = x.reshape(-1).contiguous()
        n = xv.numel()
        stream = api._stream(stream, self.root)
        f_in, m = api._oop_rows(fs[0], x, self._code, f_in, self.pm if self.pm is not None else n, self.sparsity, self.pm, n)
        if f_in is None and self._code == L.FDB_FORWARD:       # a NativeFn: f(x) at the root, as the Python f above
            f_in = torch.empty(m, dtype=torch.float64, device=self.root)
            with torch.cuda.device(self.root):
                api._native_call(fs[0], f_in, xv, stream)
        self._build(m, n)
        res = api._OopOutput(self.kind, self.sparsity, self.pn, m, self.plans[-1].dense_range()[1],
                             self.plans[0].info()["n_entries"], self.root, self.csr)
        addr, ctxs, pyfns = self._member_fns(fs, m, n, oop=True)
        api._call(self.root, pyfns, L.lib().fdb_group_jacobian_oop, self._h, addr, ctxs, xv.data_ptr(), C.byref(res.out),
                  None, api._oop_fin_ptr(f_in, self._code, m), *api._steps(relstep, absstep), float(dir),
                  C.c_void_p(stream))
        return res.result(stream)

    def close(self):
        if self._key is not None:
            super().close()
            self._key = None


class ShardedJacobian:
    """finite_difference_jacobian! with the colours of `cache.colorvec` sharded over the ranks of the default process
    group, one process per GPU (the cache must have been built with rank=, world=).

    mode="p2p" (default): no collective on the data path.  Rank 0's nzval lives in a CUDA-IPC buffer that every rank
    maps; the plans are created with shared_j, so each rank's diff+scatter kernel stores the entries it owns STRAIGHT
    into rank 0's nzval over NVLink (the literal "final gather of Jacobian columns", fused into the kernel), and the
    ranks are ordered by the device-side flag barrier of the C ABI (fdb_sync: DeviceBarrier) — no NCCL call per Jacobian.
      gather="root"     rank 0 ends with the complete J;
      gather="all"      + one NCCL broadcast of nzval (bulk, full NVLink bandwidth): every rank ends with it;
      gather="all_p2p"  every value is stored to EVERY peer by the scatter kernel (fdb_plan_set_peers).  Fine up to 4
                        GPUs, 16 ms at 8 (7 peer apertures x scattered 64-byte runs) — kept for experiments only.
    mode="nccl": pack owned entries -> all_gather -> unpack (fallback; also what the CPU/gloo tests exercise)."""

    def __init__(self, J: api.SparseMatrixCSC, cache: api.JacobianCache, n: int, device, mode: str = "p2p", group=None,
                 pre_sync: bool = True, gather: str = "all", barrier: str = "device"):
        if gather not in ("all", "root", "all_p2p"):
            raise ValueError("gather must be 'all', 'root' or 'all_p2p'")
        if barrier not in ("device", "nccl"):
            raise ValueError("barrier must be 'device' (fdb_sync) or 'nccl' (all_reduce of a flag word)")
        self.gather = gather
        if not isinstance(J, api.SparseMatrixCSC):
            raise TypeError("ShardedJacobian shards CSC Jacobians (dense / banded plans: GroupJacobian, or rank/world plans "
                            "with their own column slabs)")
        self.J, self.cache, self.n, self.device, self.group = J, cache, n, torch.device(device), group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.pre_sync = pre_sync
        self.shared = mode == "p2p" and gather in ("root", "all")
        if self.shared:
            cache._plan_kw["shared_j"] = True
        self.plan = cache.plan_for(J, cache.sparsity, cache.colorvec, n)
        self.flag = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.mode = mode
        self._peers = []
        self._root: Optional[_RootValues] = None
        self._J_run = J
        self._ipc: Optional[IpcBuffer] = None
        self.barrier: Optional[DeviceBarrier] = None
        self._barrier_kind = barrier
        if mode == "p2p":
            try:
                self._setup_p2p()
            except Exception as e:  # no IPC / no peer access: fall back to the NCCL exchange
                self.mode = "nccl"
                self._fallback_reason = repr(e)
        if self.mode == "nccl":
            cp = J.colptr.cpu().numpy() if isinstance(J.colptr, torch.Tensor) else np.asarray(J.colptr)
            cv = cache.colorvec
            cv = cv.cpu().numpy() if isinstance(cv, torch.Tensor) else np.asarray(list(cv) if isinstance(cv, range) else cv)
            self.gp = GatherPlan(entry_colors_csc(cp, cv), self.plan.color_owner(), self.world, self.device)

    def _setup_p2p(self):
        nnz = self.J.nzval.numel()
        if self.shared:
            self._root = _RootValues(self.J, self.device, self.rank, self.world, self.group)
            if self._root.ptr is not None:
                # rank 0's nzval as mapped into this process: a raw pointer (api.PeerValues), never a torch tensor
                self._J_run = api.SparseMatrixCSC(self.J.m, self.J.n, self.J.colptr, self.J.rowval,
                                                  api.PeerValues(self._root.ptr, nnz))
        else:
            self._ipc = IpcBuffer(nnz, self.device)
            self._ipc.tensor.copy_(self.J.nzval)
            self.J.nzval = self._ipc.tensor
            handles = [None] * self.world
            dist.all_gather_object(handles, self._ipc.handle(), group=self.group)
            ptrs = []
            with torch.cuda.device(self.device):
                for r, h in enumerate(handles):
                    if r == self.rank:
                        continue
                    p = C.c_void_p()
                    L.check(L.lib().fdb_ipc_open(h, C.byref(p)))
                    ptrs.append(p.value)
            self._peers = ptrs
            self.plan.set_peers(ptrs)
        if self._barrier_kind == "device":
            self.barrier = DeviceBarrier(self.device, self.group)
        ok = torch.ones(1, device=self.device)
        dist.all_reduce(ok, group=self.group)

    def _sync(self):
        if self.barrier is not None:
            self.barrier.wait()
        else:
            dist.all_reduce(self.flag, group=self.group)

    def run(self, f, x, **kw):
        if self.mode == "p2p" and self.pre_sync:
            self._sync()                                   # nobody may still be reading J (stream-ordered)
        api.finite_difference_jacobian_(self._J_run, f, x, self.cache, **kw)
        if self.mode == "p2p":
            self._sync()                                   # every rank's scatter (incl. its NVLink stores) has completed
            if self.gather == "all":
                dist.broadcast(self.J.nzval, src=0, group=self.group)
        else:
            allgather_owned(self.J.nzval, self.gp, self.rank, self.group)
        return None

    def close(self):
        torch.cuda.synchronize(self.device)
        if self._peers:
            self.plan.set_peers([])
            with torch.cuda.device(self.device):
                for p in self._peers:
                    L.lib().fdb_ipc_close(C.c_void_p(p))
            self._peers = []
        if self.barrier is not None:
            self.barrier.close()
            self.barrier = None
        if self._root is not None:
            self._root.close()
            self._root = None
            self._J_run = self.J
            return
        _barrier(self.group)
        if self._ipc is not None:
            self._ipc.free()
            self._ipc = None


# ------------------------------------------------------------------------------------------------ column-block shards
# SURVEY.md §8f row 4: problems with fewer colours than GPUs (C2: 3 colours, C3: 5) cannot be spread by colour.  A
# contiguous block of COLUMNS can: the block's entries live in a row range [r0, r1), those rows depend on an x range
# [x0, x1) (the block plus a halo), and everything the colour loop does for the block happens inside those ranges —
# with a slice-aware f! (rows [r0, r1) from x[x0:x1]) there is no exchange at all on the data path.  The only global
# quantity is the step size of each colour (norm over ALL colour-k components of x, jacobians.jl:559-561): every rank
# holds the full x and runs the K2 pass on it (fdb_color_eps), the shard plan takes the result as external step sizes.
# With the same step sizes a shard's values are bit-identical to its segment of the unsharded nzval.
def column_blocks(colptr, world: int) -> List[int]:
    """Block boundaries b[0..world] (0-based columns) balancing the number of stored entries per block."""
    cp = colptr.cpu().numpy() if isinstance(colptr, torch.Tensor) else np.asarray(colptr)
    n = len(cp) - 1
    nnz = int(cp[-1] - 1)
    bounds = [0]
    for r in range(1, world):
        target = 1 + (nnz * r) // world
        bounds.append(int(min(max(np.searchsorted(cp, target, side="left"), bounds[-1]), n)))
    bounds.append(n)
    return bounds


def block_geometry(colptr: torch.Tensor, rowval: torch.Tensor, c0: int, c1: int) -> dict:
    """Everything a column block [c0, c1) of a CSC pattern (Int64, 1-based, rows sorted inside a column) needs:
    p0, p1   0-based slot range of the block in rowval / nzval,
    r0, r1   the row range its entries touch (0-based, half-open),
    x0, x1   hull of the columns with an entry in those rows = the x slice a slice-aware f! must see (contains [c0, c1)),
    colptr_loc / rowval_loc   the block's pattern over the columns [x0, x1) and rows [r0, r1), 1-based: only the owned
             columns carry entries."""
    cp, rv = colptr, rowval
    p0, p1 = int(cp[c0]) - 1, int(cp[c1]) - 1
    seg = rv[p0:p1]
    if seg.numel() == 0:
        r0 = r1 = 0
        x0, x1 = c0, c1
    else:
        r0, r1 = int(seg.min()) - 1, int(seg.max())
        cnt = cp[1:] - cp[:-1]
        first = rv[(cp[:-1] - 1).clamp(max=max(rv.numel() - 1, 0))]
        last = rv[(cp[1:] - 2).clamp(min=0)]
        touch = (cnt > 0) & (last - 1 >= r0) & (first - 1 < r1)
        idx = torch.nonzero(touch).reshape(-1)
        x0, x1 = min(int(idx[0]), c0), max(int(idx[-1]) + 1, c1)
    j = torch.arange(x0, x1 + 1, device=cp.device)
    colptr_loc = (cp[j.clamp(c0, c1)] - p0).contiguous()
    rowval_loc = (seg - r0).contiguous()
    return dict(p0=p0, p1=p1, r0=r0, r1=r1, x0=x0, x1=x1, colptr_loc=colptr_loc, rowval_loc=rowval_loc)


class EpsPlan:
    """Step sizes of every colour for a full-length x: the K2 pass alone (fdb_eps_plan_create / fdb_color_eps)."""

    def __init__(self, n: int, colorvec, fdtype, device):
        self.device = torch.device(device)
        o = api._opts(api._fdtype_code(fdtype), api._device_index(device))
        cv_ptr, keep = api._index_ptr(colorvec)
        with torch.cuda.device(self.device):
            h = api._new_handle("fdb_eps_plan_create", int(n), cv_ptr, C.byref(o))
        self.plan = api.Plan(h.value, keep=(keep,))
        self.n_colors = self.plan.info()["n_colors"]
        self.eps = torch.zeros(max(self.n_colors, 1), dtype=torch.float64, device=self.device)

    def compute(self, x: torch.Tensor, relstep=None, absstep=None, dir=True, stream=None) -> torch.Tensor:
        api._call(self.device, (), L.lib().fdb_color_eps, self.plan.handle, x.data_ptr(), *api._steps(relstep, absstep),
                  float(dir), self.eps.data_ptr(), C.c_void_p(api._stream(stream, self.device)))
        return self.eps


class ColumnBlockJacobian:
    """The colour loop of finite_difference_jacobian! for the columns [c0, c1) of a CSC Jacobian.

    f_factory(row0, row1, x0, x1) must return the slice-aware f! (NativeFn or Python callable f(fx, x)) that computes
    rows [row0, row1) of f from x[x0:x1] (0-based, half-open).  run(x, eps) writes the block's values into
    values_ptr (default: J.nzval) at slots [p0, p1) — the same positions the unsharded call writes."""

    def __init__(self, J: api.SparseMatrixCSC, colorvec, fdtype, c0: int, c1: int, device, f_factory, *, max_batch=1,
                 use_graph=False, no_drift=False):
        self.device = torch.device(device)
        self.fdtype = fdtype
        cp = J.colptr if isinstance(J.colptr, torch.Tensor) else torch.as_tensor(np.asarray(J.colptr))
        rv = J.rowval if isinstance(J.rowval, torch.Tensor) else torch.as_tensor(np.asarray(J.rowval))
        cp, rv = cp.to(self.device), rv.to(self.device)
        self.c0, self.c1 = int(c0), int(c1)
        g = block_geometry(cp, rv, self.c0, self.c1)
        self.p0, self.p1, self.r0, self.r1, self.x0, self.x1 = g["p0"], g["p1"], g["r0"], g["r1"], g["x0"], g["x1"]
        self.m_loc, self.n_loc = self.r1 - self.r0, self.x1 - self.x0
        colptr_loc, rowval_loc = g["colptr_loc"], g["rowval_loc"]
        if isinstance(colorvec, range):
            colorvec = np.arange(colorvec.start, colorvec.stop, colorvec.step, dtype=np.int64)
        cv = colorvec if isinstance(colorvec, torch.Tensor) else torch.as_tensor(np.asarray(colorvec, dtype=np.int64))
        self.cv_loc = cv[self.x0:self.x1].to(self.device).contiguous()
        self.sub = api.SparseMatrixCSC(self.m_loc, self.n_loc, colptr_loc, rowval_loc, None)
        self.values_default = J.nzval
        self.plan = api.make_plan(self.sub, self.sub, self.cv_loc, fdtype, self.n_loc, self.device, max_batch=max_batch,
                                  use_graph=use_graph, no_drift=no_drift)
        self.f = f_factory(self.r0, self.r1, self.x0, self.x1)
        self._fn = api._as_fn(self.f, self.m_loc, self.n_loc, self.device, 1)
        self._eps_set = None

    def run(self, x: torch.Tensor, eps: torch.Tensor, values_ptr: Optional[int] = None, dir=True, stream=None):
        addr, ctx, pyfn = self._fn
        if self._eps_set != eps.data_ptr():
            L.check(L.lib().fdb_plan_set_external_eps(self.plan.handle, eps.data_ptr()))
            self._eps_set = eps.data_ptr()
        base = self.values_default.data_ptr() if values_ptr is None else int(values_ptr)
        api._call(self.device, [pyfn], L.lib().fdb_jacobian, self.plan.handle, addr, ctx, x.data_ptr() + 8 * self.x0,
                  base + 8 * self.p0, None, None, L.STEP_DEFAULT, L.STEP_DEFAULT, float(dir),
                  C.c_void_p(api._stream(stream, self.device)))


class ColumnShardedJacobian:
    """One process per GPU, every rank owns a contiguous block of columns (entry-balanced).  Every rank needs the full
    x; J stays column-sharded (gather=None: rank r's J.nzval holds its slots [p0, p1)) or is assembled on rank 0
    (gather="root": the scatter kernel stores straight into rank 0's nzval over NVLink — contiguous 16-byte stores)."""

    def __init__(self, J: api.SparseMatrixCSC, colorvec, fdtype, device, f_factory, *, gather: Optional[str] = None,
                 group=None, max_batch=1, use_graph=False):
        if gather not in (None, "root"):
            raise ValueError("gather must be None or 'root'")
        self.J, self.device, self.group, self.gather = J, torch.device(device), group, gather
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.bounds = column_blocks(J.colptr, self.world)
        self.eps_plan = EpsPlan(J.n, colorvec, fdtype, device)
        self.block = ColumnBlockJacobian(J, colorvec, fdtype, self.bounds[self.rank], self.bounds[self.rank + 1], device,
                                         f_factory, max_batch=max_batch, use_graph=use_graph)
        self.flag = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._root: Optional[_RootValues] = None
        self.barrier: Optional[DeviceBarrier] = None
        if gather == "root":
            self.barrier = DeviceBarrier(self.device, group)
            self._root = _RootValues(J, self.device, self.rank, self.world, group)
            self.block.values_default = J.nzval

    def run(self, x: torch.Tensor, dir=True):
        eps = self.eps_plan.compute(x, dir=dir)
        if self.gather == "root":
            self.barrier.wait()                               # rank 0 is done reading the previous J
        self.block.run(x, eps, values_ptr=None if self._root is None else self._root.ptr, dir=dir)
        if self.gather == "root":
            self.barrier.wait()                               # every block (incl. its NVLink stores) has completed

    def close(self):
        torch.cuda.synchronize(self.device)
        if self.barrier is not None:
            self.barrier.close()
            self.barrier = None
        if self._root is not None:
            self._root.close()
            self._root = None
        else:
            _barrier(self.group)
