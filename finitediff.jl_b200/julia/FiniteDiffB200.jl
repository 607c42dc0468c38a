# FiniteDiffB200.jl — Julia host side of the H100 drop-in for FiniteDiff.jl's coloured Jacobian path.
#
# NOT EXECUTED IN THIS REPOSITORY'S CI: the build image has no `julia` binary (SURVEY.md §8c).  The file is the binding a
# maintainer adds; the same C ABI (include/fdjac_b200.h) is exercised end-to-end through the Python/ctypes mirror
# (finitediff.jl_b200/api.py), which keeps the same names and argument meaning.  tests/test_julia_binding_cpu.py checks
# this file against the header without running it: struct layouts (field order / widths), every ccall's symbol and
# argument count, block balance.
#
# What it does: adds METHODS to FiniteDiff.finite_difference_jacobian! (src/jacobians.jl:504-514) and
# FiniteDiff.finite_difference_jvp! (src/jvp.jl:238-247) that dispatch on device arrays (CUDA.CuVector{Float64}) and forward
# the WHOLE colour loop to libfdjac_b200.so with one ccall — not the per-colour hooks (`_colorediteration!`), because a
# host round trip per colour would forfeit the device residency.  Covered: every (J, sparsity) combination the reference's
# hooks serve on this path —
#     DeviceCSC J + CSC sparsity            ext/FiniteDiffSparseArraysExt.jl:38-47 (same pattern) / :20-28 (other pattern)
#     CuMatrix J  + CSC sparsity            ext/FiniteDiffSparseArraysExt.jl:20-28
#     DeviceBanded J or CuMatrix J + Banded ext/FiniteDiffBandedMatricesExt.jl:13-27
#     DeviceTridiagonal J (structured, COO) src/iteration_utils.jl:25-32 with ArrayInterface.findstructralnz
#     DeviceDiagonal / DeviceBidiagonal J, or CuMatrix J + Diagonal / Bidiagonal / SymTridiagonal sparsity: the banded
#                                           plan on the in-matrix band (l, u) of the type (packed diagonal storage)
#     CuMatrix J + dense 0/1 prototype      src/jacobians.jl:473-488, 526-527
#     CuMatrix J, sparsity === nothing      src/jacobians.jl:548-557, 590-598 (dense column branch, colorvec quirk included)
#   for Val(:forward), Val(:central) and Val(:complex) (src/jacobians.jl:623-648), plus the JVP and the multi-GPU group,
#   and the vector -> scalar entry points on CuVector{Float64} x: finite_difference_hessian! (src/hessians.jl:202-292,
#   fdb_hessian) and finite_difference_gradient! (src/gradients.jl:390-473, the dense plan with m = 1), and the scalar-input
#   entry points through fdb_derivative: finite_difference_derivative! on CuVector{Float64} x (src/derivatives.jl:197-233)
#   and finite_difference_gradient! at a Real x into a CuVector{Float64} df (src/gradients.jl:477-533).
#   The out-of-place finite_difference_jacobian (src/jacobians.jl:240-429) and finite_difference_jvp (src/jvp.jl:133-189)
#   on CuVector{Float64} x go through fdb_jacobian_oop / fdb_jvp_oop: the trampoline copies the array f returns into the
#   slot f! would have written.
# Everything else of FiniteDiff.jl (CPU arrays, complex x, other sparsity / prototype types of the out-of-place form)
# keeps using the stock package.
module FiniteDiffB200

using FiniteDiff, SparseArrays, CUDA
using LinearAlgebra: Diagonal, Bidiagonal, SymTridiagonal, Tridiagonal
import FiniteDiff: finite_difference_jacobian!, finite_difference_jvp!, JacobianCache, JVPCache,
    finite_difference_jacobian, finite_difference_jvp,
    finite_difference_hessian!, HessianCache, finite_difference_gradient!, GradientCache, finite_difference_derivative!,
    DerivativeCache

const libfdjac = get(ENV, "FDJAC_B200_LIB", "libfdjac_b200.so")

const FDB_FORWARD, FDB_CENTRAL, FDB_COMPLEX, FDB_HCENTRAL = Cint(0), Cint(1), Cint(2), Cint(3)
const FDB_J_CSC_NZVAL, FDB_J_DENSE, FDB_J_BAND, FDB_J_SLOTS, FDB_J_BLOCK_BAND, FDB_J_DIAGONALS =
    Cint(0), Cint(1), Cint(2), Cint(3), Cint(4), Cint(5)
const FDB_STEP_DEFAULT = NaN            # relstep / absstep keyword not given (include/fdjac_b200.h)
const FDB_OOP_RAW, FDB_OOP_DENSE, FDB_OOP_SPARSE = Cint(0), Cint(1), Cint(2)

# mirror of fdb_plan_opts (include/fdjac_b200.h) — field order and widths are checked by tests/test_julia_binding_cpu.py
struct PlanOpts
    fdtype::Int32
    device::Int32
    use_current_device::Int32
    no_drift::Int32
    max_batch::Int64
    scratch_bytes::Int64
    rank::Int32
    world::Int32
    partition::Int32
    strategy::Int32
    use_graph::Int32
    shared_j::Int32
end
PlanOpts(fd; max_batch = 1, rank = 0, world = 1, use_graph = false, shared_j = false) =
    PlanOpts(fd, 0, 1, 0, max_batch, 0, rank, world, 0, 0, use_graph ? 1 : 0, shared_j ? 1 : 0)

# mirror of fdb_plan_info_t
struct PlanInfo
    m::Int64
    n::Int64
    n_entries::Int64
    j_len::Int64
    n_colors::Int64
    n_local_colors::Int64
    n_groups::Int64
    slabs::Int64
    fcalls_per_jacobian::Int64
    device_bytes::Int64
    fdtype::Int32
    jkind::Int32
    sp_kind::Int32
    color_bits::Int32
    alg_bytes_scatter::Int64
    strategy::Int32
    lanes::Int32
    mean_row_jump::Float64
    moved_bytes_scatter::Int64
    staged::Int32
    lists_resident::Int32
end

struct FdbError <: Exception
    status::Cint
    msg::String
end
function check(st::Cint)
    st == 0 && return nothing
    throw(FdbError(st, unsafe_string(ccall((:fdb_last_error, libfdjac), Cstring, ()))))
end

fdcode(::Val{:forward}) = FDB_FORWARD
fdcode(::Val{:central}) = FDB_CENTRAL
fdcode(::Val{:complex}) = FDB_COMPLEX
fdcode(::Val{T}) where {T} = FiniteDiff.fdtype_error(Float64)   # src/epsilons.jl:159-167

# ---- device-side J / sparsity wrappers: the index structure stays on the host exactly as the reference's types hold
#      it (that is what dispatch sees), the VALUES live on the device.
struct DeviceCSC
    host::SparseMatrixCSC{Float64, Int64}   # pattern (colptr / rowval)
    nzval::CuVector{Float64}                # values on the device
end
Base.size(J::DeviceCSC) = size(J.host)
Base.size(J::DeviceCSC, d) = size(J.host, d)

struct DeviceBanded                          # BandedMatrices.BandedMatrix: data[(l+u+1) x n], slot [u+r-c+1, c]
    m::Int
    n::Int
    l::Int
    u::Int
    data::CuVector{Float64}                  # (l+u+1)*n, column-major (ext/FiniteDiffBandedMatricesExt.jl:22)
end
Base.size(J::DeviceBanded) = (J.m, J.n)
Base.size(J::DeviceBanded, d) = d == 1 ? J.m : J.n

# BlockBandedMatrices.BandedBlockBandedMatrix with square blocks: the block sizes blocklengths(axes(J, 1)), the block
# bandwidths blockbandwidths(J), the sub-block bandwidths subblockbandwidths(J) and the band data on the device:
# (l+u+1)(lam+mu+1) slots per column, entry (k, j) of block (K, J) at slot (K-J+u)(lam+mu+1) + (mu+k-j) (0-based k, j)
struct DeviceBlockBanded
    blocks::Vector{Int64}
    l::Int
    u::Int
    lam::Int
    mu::Int
    data::CuVector{Float64}                  # (l+u+1)(lam+mu+1) * sum(blocks), column-major
end
Base.size(J::DeviceBlockBanded) = (sum(J.blocks), sum(J.blocks))
Base.size(J::DeviceBlockBanded, d) = sum(J.blocks)

# BlockBandedMatrices.BlockBandedMatrix with square blocks, in that package's own storage: the block sizes
# blocklengths(axes(J, 1)), the block bandwidths blockbandwidths(J) and the data vector on the device (a
# BlockBandedMatrix{Float64} whose data is a CuVector{Float64}: the plan writes pointer(data)).  Block column J
# is one column-major slab holding every row of the block rows in blockcolrange(J) (FDB_J_BLOCK_DENSE in the header).
struct DeviceBlockDense
    blocks::Vector{Int64}
    l::Int
    u::Int
    data::CuVector{Float64}                  # sum over block columns of (slab height) * (block width)
end
Base.size(J::DeviceBlockDense) = (sum(J.blocks), sum(J.blocks))
Base.size(J::DeviceBlockDense, d) = sum(J.blocks)

# A row-compressed sparse matrix on the device (the format of cuSPARSE, cuDSS and AMGX): Int64 1-based row pointer and
# columns on the device, nzval the Jacobian's values (FDB_J_CSR: J and the sparsity are this one pattern)
struct DeviceCSR
    m::Int
    n::Int
    rowptr::CuVector{Int64}                  # m + 1
    colval::CuVector{Int64}                  # nnz
    nzval::CuVector{Float64}                 # nnz
end
Base.size(J::DeviceCSR) = (J.m, J.n)
Base.size(J::DeviceCSR, d) = d == 1 ? J.m : J.n
# CUDA.jl's CuSparseMatrixCSR{Float64}: its Cint indices are widened on the device once per wrapper; nzVal is aliased, so
# the Jacobian is written in place into the matrix the solver holds
DeviceCSR(A::CUDA.CUSPARSE.CuSparseMatrixCSR{Float64}) =
    DeviceCSR(size(A, 1), size(A, 2), CuVector{Int64}(A.rowPtr), CuVector{Int64}(A.colVal), A.nzVal)

struct DeviceTridiagonal                     # LinearAlgebra.Tridiagonal(dl, d, du): one buffer [dl; d; du]
    n::Int
    buf::CuVector{Float64}                   # 3n - 2
end
Base.size(J::DeviceTridiagonal) = (J.n, J.n)
Base.size(J::DeviceTridiagonal, d) = J.n

# LinearAlgebra.Diagonal(d) / Bidiagonal(dv, ev, uplo) with the values on the device, in the packed diagonal storage of
# FDB_J_DIAGONALS (stored diagonals in ascending row-minus-column order): [d], [dv; ev] for :U, [ev; dv] for :L.  The
# LinearAlgebra types take views of the one buffer: Diagonal(view(buf, 1:n)), Bidiagonal(view(buf, 1:n),
# view(buf, n+1:2n-1), :U) or Bidiagonal(view(buf, n:2n-1), view(buf, 1:n-1), :L).
struct DeviceDiagonal
    n::Int
    buf::CuVector{Float64}                   # n
end
struct DeviceBidiagonal
    n::Int
    uplo::Symbol                             # :U or :L
    buf::CuVector{Float64}                   # 2n - 1
end
Base.size(J::Union{DeviceDiagonal, DeviceBidiagonal}) = (J.n, J.n)
Base.size(J::Union{DeviceDiagonal, DeviceBidiagonal}, d) = J.n

# the in-matrix band (l, u) that is the entry set of each type (ArrayInterface.findstructralnz)
bands(::Union{DeviceDiagonal, Diagonal}) = (0, 0)
bands(J::Union{DeviceBidiagonal, Bidiagonal}) = (J.uplo == :U || J.uplo == 'U') ? (0, 1) : (1, 0)
bands(::SymTridiagonal) = (1, 1)

# ArrayInterface.matrix_colors closed forms: all 1 (Diagonal), cycle 1:2 (Bidiagonal), cycle 1:3 (SymTridiagonal)
function matrix_colors(J::Union{DeviceDiagonal, DeviceBidiagonal, Diagonal, Bidiagonal, SymTridiagonal})
    n = size(J, 2)
    l, u = bands(J)
    out = CuVector{Int64}(undef, max(n, 1))
    GC.@preserve out begin
        check(ccall((:fdb_matrix_colors_banded, libfdjac), Cint, (Int64, Int64, Int64, CuPtr{Int64}, Ptr{Cvoid}),
            n, l, u, pointer(out), CUDA.stream().handle))
    end
    out[1:n]
end

# ArrayInterface.findstructralnz(::Tridiagonal): band by band (order is irrelevant to the result); slots into [dl; d; du]
function tridiagonal_structure(n::Int)
    rows = vcat(collect(Int64, 2:n), collect(Int64, 1:n), collect(Int64, 1:(n - 1)))
    cols = vcat(collect(Int64, 1:(n - 1)), collect(Int64, 1:n), collect(Int64, 2:n))
    slots = collect(Int64, 1:(3n - 2))
    rows, cols, slots
end

# src/jacobians.jl:473-488 — column-major scan of a dense 0/1 prototype
function dense_prototype_structure(A::AbstractMatrix)
    rows, cols = Int64[], Int64[]
    for j in axes(A, 2), i in axes(A, 1)
        if !iszero(A[i, j])
            push!(rows, i)
            push!(cols, j)
        end
    end
    rows, cols
end

# ---- plans: the per-(pattern, colorvec, fdtype) state the reference rebuilds on every call (jacobians.jl:515-535).
# Cached per index array: a WeakKeyDict keyed on the (mutable) anchor array of the pattern — when the caller drops the
# pattern the entry and its plans go away (finalizer -> fdb_plan_destroy); nothing is pinned forever.
mutable struct Plan
    handle::Ptr{Cvoid}
    roots::Any                     # host index arrays the plan was built from (kept alive for the plan's lifetime)
    function Plan(h, roots = nothing)
        p = new(h, roots)
        finalizer(q -> ccall((:fdb_plan_destroy, libfdjac), Cint, (Ptr{Cvoid},), q.handle), p)
        p
    end
end
const PLANS = WeakKeyDict{Any, Dict{Any, Plan}}()
const PLANS_LOCK = ReentrantLock()

function cached_plan(make::Function, anchor, key)
    lock(PLANS_LOCK) do
        d = get!(() -> Dict{Any, Plan}(), PLANS, anchor)
        get!(make, d, key)
    end
end

# colorvec as the ABI wants it: (pointer, root).  The ROOT must stay referenced (GC.@preserve) across the ccall:
# a freshly collected Vector is returned together with its pointer, never a pointer to a temporary.
function color_arg(cv::AbstractUnitRange, n::Integer)
    (first(cv) == 1 && length(cv) == n) && return (Ptr{Int64}(C_NULL), nothing)      # NULL => 1:n (jacobians.jl:16)
    v = collect(Int64, cv)
    (pointer(v), v)
end
function color_arg(cv::Vector{Int64}, n::Integer)
    (pointer(cv), cv)
end
function color_arg(cv::AbstractVector{<:Integer}, n::Integer)
    v = collect(Int64, cv)
    (pointer(v), v)
end
color_key(cv::AbstractUnitRange) = (:range, first(cv), last(cv))
color_key(cv) = (:vec, objectid(cv), length(cv))

function info(plan::Plan)
    r = Ref{PlanInfo}()
    check(ccall((:fdb_plan_info, libfdjac), Cint, (Ptr{Cvoid}, Ref{PlanInfo}), plan.handle, r))
    r[]
end

# sparsity::SparseMatrixCSC — J is a DeviceCSC (nzval slots) or a dense CuMatrix (ldJ)
function plan_csc(sp::SparseMatrixCSC{Float64, Int64}, Jhost, ldJ::Integer, colorvec, fd::Cint; kw...)
    jk = Jhost === nothing ? FDB_J_DENSE : FDB_J_CSC_NZVAL
    same = Jhost === nothing || Jhost === sp || (Jhost.colptr === sp.colptr && Jhost.rowval === sp.rowval)
    key = (:csc, objectid(sp.rowval), same ? 0 : objectid(Jhost.rowval), jk, ldJ, color_key(colorvec), fd, values(kw))
    cached_plan(sp.colptr, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        m, n = size(sp)
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve sp Jhost croot begin
            check(ccall((:fdb_plan_create_csc, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Cint, Ptr{Int64}, Ptr{Int64}, Int64, Ptr{Int64}, Ref{PlanOpts}),
                h, m, n, pointer(sp.colptr), pointer(sp.rowval), jk,
                same ? Ptr{Int64}(C_NULL) : pointer(Jhost.colptr), same ? Ptr{Int64}(C_NULL) : pointer(Jhost.rowval), ldJ,
                cptr, opts))
        end
        Plan(h[], (sp, Jhost, croot))
    end
end

# structural-nonzero lists (Tridiagonal / dense prototype): generic hook src/iteration_utils.jl:25-32
# `structure()` returns (rows, cols, slots-or-nothing); it runs only when the plan is not cached yet, so a cached call does
# no O(nnz) host work (the reference rebuilds these lists on every call, jacobians.jl:522-528)
function plan_coo(structure::Function, anchor, m::Integer, n::Integer, tag, jk::Cint, ld_or_len::Integer, colorvec, fd::Cint; kw...)
    key = (:coo, m, n, tag, jk, ld_or_len, color_key(colorvec), fd, values(kw))
    cached_plan(anchor, key) do
        rows, cols, slots = structure()
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve rows cols slots croot begin
            check(ccall((:fdb_plan_create_coo, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Cint, Ptr{Int64}, Int64, Ptr{Int64}, Ref{PlanOpts}),
                h, m, n, length(rows), pointer(rows), pointer(cols), jk,
                slots === nothing ? Ptr{Int64}(C_NULL) : pointer(slots), ld_or_len, cptr, opts))
        end
        Plan(h[], (rows, cols, slots, croot))
    end
end

# sparsity::BandedMatrix(l, u): ext/FiniteDiffBandedMatricesExt.jl:13-27 (whole band)
function plan_banded(anchor, m::Integer, n::Integer, l::Integer, u::Integer, jk::Cint, ldJ::Integer, colorvec, fd::Cint; kw...)
    key = (:banded, m, n, l, u, jk, ldJ, color_key(colorvec), fd, values(kw))
    cached_plan(anchor, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve croot begin
            check(ccall((:fdb_plan_create_banded, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, Int64, Int64, Cint, Int64, Ptr{Int64}, Ref{PlanOpts}),
                h, m, n, l, u, jk, ldJ, cptr, opts))
        end
        Plan(h[], croot)
    end
end

# sparsity::BandedBlockBandedMatrix, J the same structure: ext/FiniteDiffBlockBandedMatricesExt.jl:16-42 as a closed form
# (no entry lists on the host)
function plan_block_banded(J::DeviceBlockBanded, colorvec, fd::Cint; kw...)
    key = (:block_banded, J.blocks, J.l, J.u, J.lam, J.mu, length(J.data), color_key(colorvec), fd, values(kw))
    cached_plan(J.data, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, size(J, 2))
        blocks = J.blocks
        GC.@preserve blocks croot begin
            check(ccall((:fdb_plan_create_block_banded, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Ptr{Int64}, Int64, Int64, Int64, Int64, Int64, Ptr{Int64}, Ref{PlanOpts}),
                h, length(blocks), pointer(blocks), J.l, J.u, J.lam, J.mu, length(J.data), cptr, opts))
        end
        Plan(h[], (blocks, croot))
    end
end

# sparsity::BlockBandedMatrix, J the same structure: ext/FiniteDiffBlockBandedMatricesExt.jl:44-68 as a closed form
# over BlockBandedMatrices' storage (no entry lists on the host)
function plan_block_dense(J::DeviceBlockDense, colorvec, fd::Cint; kw...)
    key = (:block_dense, J.blocks, J.l, J.u, length(J.data), color_key(colorvec), fd, values(kw))
    cached_plan(J.data, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, size(J, 2))
        blocks = J.blocks
        GC.@preserve blocks croot begin
            check(ccall((:fdb_plan_create_block_dense, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Ptr{Int64}, Int64, Int64, Int64, Ptr{Int64}, Ref{PlanOpts}),
                h, length(blocks), pointer(blocks), J.l, J.u, length(J.data), cptr, opts))
        end
        Plan(h[], (blocks, croot))
    end
end

# J and sparsity one CSR pattern: the nzval scatter, indices read from the device (ext/FiniteDiffSparseArraysExt.jl:20-28 on a
# row-compressed target)
function plan_csr(J::DeviceCSR, colorvec, fd::Cint; kw...)
    key = (:csr, J.m, J.n, objectid(J.rowptr), objectid(J.colval), color_key(colorvec), fd, values(kw))
    cached_plan(J.nzval, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, J.n)
        rowptr, colval = J.rowptr, J.colval
        GC.@preserve rowptr colval croot begin
            check(ccall((:fdb_plan_create_csr, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Ptr{Int64}, Ref{PlanOpts}),
                h, J.m, J.n, pointer(rowptr), pointer(colval), cptr, opts))
        end
        Plan(h[], (rowptr, colval, croot))
    end
end

# sparsity === nothing: dense column branch; a non-default colorvec reproduces jacobians.jl:547-557 as written
function plan_dense(anchor, m::Integer, n::Integer, ldJ::Integer, colorvec, fd::Cint; kw...)
    key = (:dense, m, n, ldJ, color_key(colorvec), fd, values(kw))
    cached_plan(anchor, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve croot begin
            check(ccall((:fdb_plan_create_dense_colorvec, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, Int64, Ptr{Int64}, Ref{PlanOpts}), h, m, n, ldJ, cptr, opts))
        end
        Plan(h[], croot)
    end
end

# ---- user function: a Julia closure f!(fx::CuVector, x::CuVector) behind the fdb_fn C signature
# int f(void* ctx, double* d_fx, const double* d_x, int64 batch, int64 ldfx, int64 ldx, void* stream)
mutable struct FnState
    f::Any
    m::Int
    n::Int
    err::Any
end

function f_trampoline(ctx::Ptr{Cvoid}, fx::CuPtr{Float64}, x::CuPtr{Float64}, batch::Int64, ldfx::Int64, ldx::Int64,
        stream::Ptr{Cvoid})::Cint
    st = unsafe_pointer_to_objref(ctx)::FnState
    try
        for b in 0:(batch - 1)          # plans are created with max_batch = 1 for plain closures
            fxv = unsafe_wrap(CuArray, fx + b * ldfx * sizeof(Float64), st.m)
            xv = unsafe_wrap(CuArray, x + b * ldx * sizeof(Float64), st.n)
            st.f(fxv, xv)               # must only enqueue on the task-local CUDA.jl stream (== `stream`)
        end
        return Cint(0)
    catch err
        st.err = err                    # never unwind through C: report, rethrow on the Julia side
        return Cint(1)
    end
end

# complex-step callback (fdb_fn_c): complex128 arrays, ld* count COMPLEX elements
function f_trampoline_c(ctx::Ptr{Cvoid}, fx::CuPtr{ComplexF64}, x::CuPtr{ComplexF64}, batch::Int64, ldfx::Int64, ldx::Int64,
        stream::Ptr{Cvoid})::Cint
    st = unsafe_pointer_to_objref(ctx)::FnState
    try
        for b in 0:(batch - 1)
            fxv = unsafe_wrap(CuArray, fx + b * ldfx * sizeof(ComplexF64), st.m)
            xv = unsafe_wrap(CuArray, x + b * ldx * sizeof(ComplexF64), st.n)
            st.f(fxv, xv)
        end
        return Cint(0)
    catch err
        st.err = err
        return Cint(1)
    end
end

stepval(::Nothing) = FDB_STEP_DEFAULT
stepval(v::Real) = Float64(v)

# the one place the hot path is entered: fdb_jacobian / fdb_jacobian_complex on the current CUDA.jl stream
function run_plan!(plan::Plan, jvals::CuArray{Float64}, f, x::CuVector{Float64}, fx, f_in, m::Integer, fdtype, relstep, absstep, dir)
    st = FnState(f, m, length(x), nothing)
    rc = Cint(0)
    if fdtype == Val(:complex)
        cf = @cfunction(f_trampoline_c, Cint, (Ptr{Cvoid}, CuPtr{ComplexF64}, CuPtr{ComplexF64}, Int64, Int64, Int64, Ptr{Cvoid}))
        GC.@preserve st x jvals begin
            rc = ccall((:fdb_jacobian_complex, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Ptr{Cvoid}),
                plan.handle, cf, pointer_from_objref(st), pointer(x), pointer(jvals), CUDA.stream().handle)
        end
    else
        cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
        GC.@preserve st x jvals fx f_in begin
            rc = ccall((:fdb_jacobian, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64},
                    Float64, Float64, Float64, Ptr{Cvoid}),
                plan.handle, cf, pointer_from_objref(st), pointer(x), pointer(jvals),
                (fx === nothing || eltype(fx) != Float64) ? CU_NULL : pointer(fx),
                f_in === nothing ? CU_NULL : pointer(f_in), stepval(relstep), stepval(absstep), Float64(dir),
                CUDA.stream().handle)
        end
    end
    st.err === nothing || throw(st.err)     # an exception inside f! propagates like in the reference
    check(rc)
    nothing                                  # jacobians.jl:652
end

const DeviceJ = Union{DeviceCSC, DeviceCSR, DeviceBanded, DeviceBlockBanded, DeviceBlockDense, DeviceTridiagonal, DeviceDiagonal, DeviceBidiagonal,
    CuMatrix{Float64}}

ld(J::CuMatrix) = max(stride(J, 2), size(J, 1), 1)

# dispatch on (typeof(J), typeof(sparsity)) — what _use_findstructralnz / _use_sparseCSC_common_sparsity / the ext
# methods decide in the reference (jacobians.jl:522-535)
function plan_for(J::DeviceCSC, sp, colorvec, fd)
    sph = sp isa DeviceCSC ? sp.host : sp
    sph isa SparseMatrixCSC || throw(ArgumentError("a DeviceCSC Jacobian needs a SparseMatrixCSC sparsity"))
    (plan_csc(sph, J.host, 0, colorvec, fd), J.nzval)
end
function plan_for(J::DeviceCSR, sp, colorvec, fd)
    (sp === J || (sp isa DeviceCSR && sp.rowptr === J.rowptr && sp.colval === J.colval)) ||
        throw(ArgumentError("not built: a DeviceCSR Jacobian with another sparsity than its own pattern"))
    (plan_csr(J, colorvec, fd), J.nzval)
end
function plan_for(J::DeviceBanded, sp, colorvec, fd)
    (sp isa DeviceBanded && (sp.l, sp.u) == (J.l, J.u)) || throw(ArgumentError("J and sparsity must have the same bandwidths"))
    (plan_banded(J.data, J.m, J.n, J.l, J.u, FDB_J_BAND, 0, colorvec, fd), J.data)
end
function plan_for(J::DeviceBlockBanded, sp, colorvec, fd)
    (sp isa DeviceBlockBanded && (sp.blocks, sp.l, sp.u, sp.lam, sp.mu) == (J.blocks, J.l, J.u, J.lam, J.mu)) ||
        throw(ArgumentError("J and sparsity must have the same block structure"))
    (plan_block_banded(J, colorvec, fd), J.data)
end
function plan_for(J::DeviceBlockDense, sp, colorvec, fd)
    (sp isa DeviceBlockDense && (sp.blocks, sp.l, sp.u) == (J.blocks, J.l, J.u)) ||
        throw(ArgumentError("J and sparsity must have the same block structure"))
    (plan_block_dense(J, colorvec, fd), J.data)
end
function plan_for(J::DeviceTridiagonal, sp, colorvec, fd)
    (plan_coo(() -> tridiagonal_structure(J.n), J.buf, J.n, J.n, :tridiagonal, FDB_J_SLOTS, 3 * J.n - 2, colorvec, fd), J.buf)
end
# Diagonal / Bidiagonal J: the banded plan into the packed diagonal storage; the sparsity is the same type or J itself
function plan_for(J::Union{DeviceDiagonal, DeviceBidiagonal}, sp, colorvec, fd)
    (typeof(sp) == typeof(J) && size(sp) == size(J) && bands(sp) == bands(J)) ||
        throw(ArgumentError("a $(typeof(J)) Jacobian needs a sparsity of the same type, size and bands"))
    l, u = bands(J)
    (plan_banded(J.buf, J.n, J.n, l, u, FDB_J_DIAGONALS, length(J.buf), colorvec, fd), J.buf)
end
function plan_for(J::CuMatrix{Float64}, sp, colorvec, fd)
    m, n = size(J)
    if sp === nothing                                                   # jacobians.jl:548-557
        return (plan_dense(J, m, n, ld(J), colorvec, fd), J)
    elseif sp isa DeviceCSC || sp isa SparseMatrixCSC                   # ext/..SparseArraysExt.jl:20-28
        sph = sp isa DeviceCSC ? sp.host : sp
        return (plan_csc(sph, nothing, ld(J), colorvec, fd), J)
    elseif sp isa DeviceBanded                                          # ext/..BandedMatricesExt.jl:13-27, dense target
        return (plan_banded(J, m, n, sp.l, sp.u, FDB_J_DENSE, ld(J), colorvec, fd), J)
    elseif sp isa DeviceTridiagonal
        return (plan_coo(J, m, n, :tridiagonal, FDB_J_DENSE, ld(J), colorvec, fd) do
                rows, cols, _ = tridiagonal_structure(sp.n)
                (rows, cols, nothing)
            end, J)
    elseif sp isa Union{Diagonal, Bidiagonal, SymTridiagonal, DeviceDiagonal, DeviceBidiagonal}
        # the type's structure only (its band), not its values; LinearAlgebra.Tridiagonal keeps the prototype method below
        (m, n) == size(sp) || throw(DimensionMismatch("size(J) != size(sparsity)"))
        l, u = bands(sp)
        return (plan_banded(J, m, n, l, u, FDB_J_DENSE, ld(J), colorvec, fd), J)
    elseif sp isa AbstractMatrix                                        # dense 0/1 prototype, jacobians.jl:526-527
        # keyed on the prototype's identity: editing it in place needs a new array (as for every cached pattern)
        return (plan_coo(J, m, n, (:prototype, objectid(sp)), FDB_J_DENSE, ld(J), colorvec, fd) do
                rows, cols = dense_prototype_structure(sp)
                (rows, cols, nothing)
            end, J)
    end
    throw(ArgumentError("unsupported sparsity type $(typeof(sp))"))
end

"""
    finite_difference_jacobian!(J, f!, x::CuVector{Float64}, cache::JacobianCache, f_in = nothing;
                                relstep, absstep, colorvec, sparsity, dir)

Same signature and keyword meaning as `src/jacobians.jl:504-514`.  `J` is a `DeviceCSC`, `DeviceBanded`,
`DeviceBlockBanded`, `DeviceBlockDense`, `DeviceTridiagonal`, `DeviceDiagonal`, `DeviceBidiagonal` or a dense `CuMatrix{Float64}`; `x`,
`cache.fx`, `f_in` are `CuVector{Float64}`.
`relstep` / `absstep` left at their defaults are passed as FDB_STEP_DEFAULT; explicit values (0 included) as given.
"""
function finite_difference_jacobian!(J::DeviceJ, f, x::CuVector{Float64},
        cache::JacobianCache{T1, T2, T3, T4, cType, sType, fdtype, returntype}, f_in = nothing;
        relstep = nothing, absstep = relstep,
        colorvec = cache.colorvec, sparsity = cache.sparsity, dir = true) where {T1, T2, T3, T4, cType, sType, fdtype, returntype}
    size(J, 2) == length(x) || throw(DimensionMismatch("size(J,2) != length(x)"))
    plan, jvals = plan_for(J, sparsity, colorvec, fdcode(fdtype))
    run_plan!(plan, jvals, f, x, cache.fx, f_in, size(J, 1), fdtype, relstep, absstep, dir)
end

# ---- JVP: finite_difference_jvp!(jvp, f, x, v, cache::JVPCache, f_in; relstep, absstep, dir)   src/jvp.jl:238-274
const JVP_PLANS = Dict{Tuple{Int, Int, Cint}, Plan}()

function jvp_plan(m::Integer, n::Integer, fd::Cint)
    lock(PLANS_LOCK) do
        get!(JVP_PLANS, (Int(m), Int(n), fd)) do
            h = Ref{Ptr{Cvoid}}(C_NULL)
            opts = Ref(PlanOpts(fd))
            check(ccall((:fdb_jvp_plan_create, libfdjac), Cint, (Ref{Ptr{Cvoid}}, Int64, Int64, Ref{PlanOpts}), h, m, n, opts))
            Plan(h[])
        end
    end
end

function finite_difference_jvp!(jvp::CuVector{Float64}, f, x::CuVector{Float64}, v::CuVector{Float64},
        cache::JVPCache{X1, FX1, fdtype}, f_in = nothing;
        relstep = nothing, absstep = relstep, dir = true) where {X1, FX1, fdtype}
    fdtype == Val(:complex) && error("finite_difference_jvp doesn't support :complex-mode finite diff")   # jvp.jl:248-250
    plan = jvp_plan(length(jvp), length(x), fdcode(fdtype))
    st = FnState(f, length(jvp), length(x), nothing)
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve st jvp x v cache f_in begin
        rc = ccall((:fdb_jvp, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64},
                CuPtr{Float64}, Float64, Float64, Float64, Ptr{Cvoid}),
            plan.handle, cf, pointer_from_objref(st), pointer(jvp), pointer(x), pointer(v), pointer(cache.x1), pointer(cache.fx1),
            f_in === nothing ? CU_NULL : pointer(f_in), stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
    end
    st.err === nothing || throw(st.err)
    check(rc)
    nothing
end

# ---- vector -> scalar: Hessian (src/hessians.jl:202-292) and gradient (src/gradients.jl:390-473) -------------------------
# f(x) returns a scalar; the trampoline stores it at fx[b*ldfx] with a device-side fill (no host synchronisation when the
# value is already on the device or a plain Number)
scalar_f(f) = (fx, xv) -> (fx .= f(xv); nothing)

function hessian_plan(H::CuMatrix{Float64}, n::Integer, ldH::Integer; kw...)
    cached_plan(H, (:hessian, n, ldH, values(kw))) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(FDB_HCENTRAL; kw...))
        check(ccall((:fdb_hessian_plan_create, libfdjac), Cint, (Ref{Ptr{Cvoid}}, Int64, Int64, Ref{PlanOpts}), h, n, ldH, opts))
        Plan(h[], nothing)
    end
end

function finite_difference_hessian!(H::CuMatrix{Float64}, f, x::CuVector{Float64}, cache::HessianCache{T, fdtype, inplace};
        relstep = nothing, absstep = relstep) where {T, fdtype, inplace}
    @assert fdtype == Val(:hcentral)                                   # hessians.jl:206
    n = length(x)
    size(H) == (n, n) || throw(DimensionMismatch("H must be $n x $n"))
    plan = hessian_plan(H, n, ld(H))
    st = FnState(scalar_f(f), 1, n, nothing)
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve st H x begin
        rc = ccall((:fdb_hessian, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, Float64, Float64, Ptr{Cvoid}),
            plan.handle, cf, pointer_from_objref(st), pointer(x), pointer(H), CU_NULL, stepval(relstep), stepval(absstep),
            CUDA.stream().handle)
    end
    st.err === nothing || throw(st.err)
    check(rc)
    H                                                                  # both triangles written (copytri!, :291)
end

finite_difference_hessian!(H::CuMatrix{Float64}, f, x::CuVector{Float64}, fdtype = Val(:hcentral), inplace = Val(true);
        relstep = nothing, absstep = relstep) =
    finite_difference_hessian!(H, f, x, HessianCache(x, fdtype, inplace); relstep = relstep, absstep = absstep)

# the gradient is the dense column branch with m = 1 (gradients.jl:408-468 vs jacobians.jl:548-557, 590-598, 625-631):
# df is J (1 x n, ldJ = 1); cache.fx, when given, is f_in (:410)
function finite_difference_gradient!(df::CuVector{Float64}, f, x::CuVector{Float64},
        cache::GradientCache{T1, T2, T3, T4, fdtype, returntype, inplace};
        relstep = nothing, absstep = relstep, dir = true) where {T1, T2, T3, T4, fdtype, returntype, inplace}
    n = length(x)
    length(df) == n || throw(DimensionMismatch("length(df) != length(x)"))
    plan = plan_dense(df, 1, n, 1, 1:n, fdcode(fdtype))
    f_in = (fdtype == Val(:forward) && cache.fx !== nothing) ? CuArray(Float64[cache.fx]) : nothing
    run_plan!(plan, df, scalar_f(f), x, nothing, f_in, 1, fdtype, relstep, absstep, dir)
    df
end

finite_difference_gradient!(df::CuVector{Float64}, f, x::CuVector{Float64}, fdtype::Union{Type, Val} = Val(:central);
        relstep = nothing, absstep = relstep, dir = true) =
    finite_difference_gradient!(df, f, x, GradientCache(df, x, fdtype); relstep = relstep, absstep = absstep, dir = dir)

# ---- scalar input per step size: finite_difference_derivative! (src/derivatives.jl:197-233) and the scalar -> vector
#      finite_difference_gradient! (src/gradients.jl:477-533), both through fdb_derivative
# the derivative's f is a scalar function applied elementwise (the plan's callback has m = n)
elementwise_f(f) = (fx, xv) -> (fx .= f.(xv); nothing)

# scalar -> vector callback: point b is ONE device double (complex: one ComplexF64), read back for the Number the reference
# passes to f(fx, t).  The read synchronises the stream, so this callback is not for use_graph plans.
function tvec_trampoline(ctx::Ptr{Cvoid}, fx::CuPtr{Float64}, x::CuPtr{Float64}, batch::Int64, ldfx::Int64, ldx::Int64,
        stream::Ptr{Cvoid})::Cint
    st = unsafe_pointer_to_objref(ctx)::FnState
    try
        for b in 0:(batch - 1)
            fxv = unsafe_wrap(CuArray, fx + b * ldfx * sizeof(Float64), st.m)
            t = Array(unsafe_wrap(CuArray, x + b * ldx * sizeof(Float64), 1))[1]
            st.f(fxv, t)
        end
        return Cint(0)
    catch err
        st.err = err
        return Cint(1)
    end
end

function tvec_trampoline_c(ctx::Ptr{Cvoid}, fx::CuPtr{ComplexF64}, x::CuPtr{ComplexF64}, batch::Int64, ldfx::Int64,
        ldx::Int64, stream::Ptr{Cvoid})::Cint
    st = unsafe_pointer_to_objref(ctx)::FnState
    try
        for b in 0:(batch - 1)
            fxv = unsafe_wrap(CuArray, fx + b * ldfx * sizeof(ComplexF64), st.m)
            t = Array(unsafe_wrap(CuArray, x + b * ldx * sizeof(ComplexF64), 1))[1]
            st.f(fxv, t)
        end
        return Cint(0)
    catch err
        st.err = err
        return Cint(1)
    end
end

function derivative_plan(anchor, scalar_input::Bool, len::Integer, fd::Cint; kw...)
    cached_plan(anchor, (scalar_input ? :scalar_gradient : :derivative, len, fd, values(kw))) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd; kw...))
        if scalar_input
            check(ccall((:fdb_scalar_gradient_plan_create, libfdjac), Cint, (Ref{Ptr{Cvoid}}, Int64, Ref{PlanOpts}), h, len, opts))
        else
            check(ccall((:fdb_derivative_plan_create, libfdjac), Cint, (Ref{Ptr{Cvoid}}, Int64, Ref{PlanOpts}), h, len, opts))
        end
        Plan(h[], nothing)
    end
end

function run_derivative!(plan::Plan, df::CuVector{Float64}, st::FnState, x::CuVector{Float64}, fx, fdtype, relstep,
        absstep, dir, scalar_input::Bool)
    rc = Cint(0)
    if fdtype == Val(:complex)
        cf = scalar_input ?
            @cfunction(tvec_trampoline_c, Cint, (Ptr{Cvoid}, CuPtr{ComplexF64}, CuPtr{ComplexF64}, Int64, Int64, Int64, Ptr{Cvoid})) :
            @cfunction(f_trampoline_c, Cint, (Ptr{Cvoid}, CuPtr{ComplexF64}, CuPtr{ComplexF64}, Int64, Int64, Int64, Ptr{Cvoid}))
        GC.@preserve st x df begin
            rc = ccall((:fdb_derivative_complex, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Ptr{Cvoid}),
                plan.handle, cf, pointer_from_objref(st), pointer(df), pointer(x), CUDA.stream().handle)
        end
    else
        cf = scalar_input ?
            @cfunction(tvec_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid})) :
            @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
        GC.@preserve st x df fx begin
            rc = ccall((:fdb_derivative, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, Float64, Float64,
                    Float64, Ptr{Cvoid}),
                plan.handle, cf, pointer_from_objref(st), pointer(df), pointer(x), fx === nothing ? CU_NULL : pointer(fx),
                stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
        end
    end
    st.err === nothing || throw(st.err)
    check(rc)
    df
end

# cache.fx is read in forward mode only (the DerivativeCache constructor already drops it otherwise, :67-73); the
# epsilon array is neither read nor written on this path
function finite_difference_derivative!(df::CuVector{Float64}, f, x::CuVector{Float64},
        cache::DerivativeCache{T1, T2, fdtype, returntype}; relstep = nothing, absstep = relstep,
        dir = true) where {T1, T2, fdtype, returntype}
    n = length(x)
    length(df) == n || throw(DimensionMismatch("length(df) != length(x)"))
    plan = derivative_plan(df, false, n, fdcode(fdtype))
    fx = (fdtype == Val(:forward) && cache.fx isa CuVector{Float64}) ? cache.fx : nothing
    run_derivative!(plan, df, FnState(elementwise_f(f), n, n, nothing), x, fx, fdtype, relstep, absstep, dir, false)
end

finite_difference_derivative!(df::CuVector{Float64}, f, x::CuVector{Float64}, fdtype::Union{Type, Val} = Val(:central),
        returntype = eltype(x), fx = nothing, epsilon = nothing; relstep = nothing, absstep = relstep) =
    finite_difference_derivative!(df, f, x, DerivativeCache(x, fx, epsilon, fdtype, returntype); relstep = relstep,
        absstep = absstep)

# the scalar t is staged into ONE device slot per cache (anchored on its c1 array, or on df when the cache has none), so
# repeated calls pass the same device pointer
const T_SLOTS = WeakKeyDict{Any, CuVector{Float64}}()

function finite_difference_gradient!(df::CuVector{Float64}, f, x::Real,
        cache::GradientCache{T1, T2, T3, T4, fdtype, returntype, inplace};
        relstep = nothing, absstep = relstep, dir = true) where {T1, T2, T3, T4, fdtype, returntype, inplace}
    m = length(df)
    anchor = cache.c1 isa CuArray ? cache.c1 : df
    t = lock(PLANS_LOCK) do
        get!(() -> CuVector{Float64}(undef, 1), T_SLOTS, anchor)
    end
    fill!(t, Float64(x))
    plan = derivative_plan(anchor, true, m, fdcode(fdtype))
    fx = (fdtype == Val(:forward) && cache.fx isa CuVector{Float64}) ? cache.fx : nothing     # gradients.jl:501-502
    run_derivative!(plan, df, FnState(f, m, 1, nothing), t, fx, fdtype, relstep, absstep, dir, true)
end

finite_difference_gradient!(df::CuVector{Float64}, f, x::Real, fdtype::Union{Type, Val} = Val(:central);
        relstep = nothing, absstep = relstep, dir = true) =
    finite_difference_gradient!(df, f, x, GradientCache(df, x, fdtype); relstep = relstep, absstep = absstep, dir = dir)

# ---- several GPUs from ONE call: fdb_group_* (colours / dense column blocks partitioned over `devices`; devices[1] is the
#      root and owns x, J, cache.fx; every member's scatter kernel stores its entries straight into the root's J).
mutable struct Group
    handle::Ptr{Cvoid}
    n::Int
    roots::Any
    function Group(h, n, roots)
        g = new(h, n, roots)
        finalizer(q -> ccall((:fdb_group_destroy, libfdjac), Cint, (Ptr{Cvoid},), q.handle), g)
        g
    end
end

function group_csc(J::DeviceCSC, colorvec, fdtype, devices::Vector{Cint}; kw...)
    sp = J.host
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    m, n = size(sp)
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve sp croot devices begin
        check(ccall((:fdb_group_create_csc, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Cint, Ptr{Int64}, Ptr{Int64}, Int64, Ptr{Int64},
                Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, pointer(sp.colptr), pointer(sp.rowval), FDB_J_CSC_NZVAL,
            Ptr{Int64}(C_NULL), Ptr{Int64}(C_NULL), 0, cptr, opts))
    end
    Group(h[], length(devices), (sp, croot))
end

function group_banded(J::DeviceBanded, colorvec, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, J.n)
    GC.@preserve croot devices begin
        check(ccall((:fdb_group_create_banded, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Int64, Int64, Cint, Int64, Ptr{Int64}, Ref{PlanOpts}),
            h, length(devices), pointer(devices), J.m, J.n, J.l, J.u, FDB_J_BAND, 0, cptr, opts))
    end
    Group(h[], length(devices), croot)
end

# Diagonal / Bidiagonal J: members write disjoint column sets of the packed diagonals, with no zero fill
function group_banded(J::Union{DeviceDiagonal, DeviceBidiagonal}, colorvec, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, J.n)
    l, u = bands(J)
    GC.@preserve croot devices begin
        check(ccall((:fdb_group_create_banded, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Int64, Int64, Cint, Int64, Ptr{Int64}, Ref{PlanOpts}),
            h, length(devices), pointer(devices), J.n, J.n, l, u, FDB_J_DIAGONALS, length(J.buf), cptr, opts))
    end
    Group(h[], length(devices), croot)
end

function group_block_banded(J::DeviceBlockBanded, colorvec, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, size(J, 2))
    blocks = J.blocks
    GC.@preserve blocks croot devices begin
        check(ccall((:fdb_group_create_block_banded, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Ptr{Int64}, Int64, Int64, Int64, Int64, Int64, Ptr{Int64}, Ref{PlanOpts}),
            h, length(devices), pointer(devices), length(blocks), pointer(blocks), J.l, J.u, J.lam, J.mu, length(J.data),
            cptr, opts))
    end
    Group(h[], length(devices), (blocks, croot))
end

function group_block_dense(J::DeviceBlockDense, colorvec, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, size(J, 2))
    blocks = J.blocks
    GC.@preserve blocks croot devices begin
        check(ccall((:fdb_group_create_block_dense, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Ptr{Int64}, Int64, Int64, Int64, Ptr{Int64}, Ref{PlanOpts}),
            h, length(devices), pointer(devices), length(blocks), pointer(blocks), J.l, J.u, length(J.data), cptr, opts))
    end
    Group(h[], length(devices), (blocks, croot))
end

function group_csr(J::DeviceCSR, colorvec, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, J.n)
    rowptr, colval = J.rowptr, J.colval
    GC.@preserve rowptr colval croot devices begin
        check(ccall((:fdb_group_create_csr, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Ptr{Int64}, Ref{PlanOpts}),
            h, length(devices), pointer(devices), J.m, J.n, pointer(rowptr), pointer(colval), cptr, opts))
    end
    Group(h[], length(devices), (rowptr, colval, croot))
end

function group_dense(J::CuMatrix{Float64}, fdtype, devices::Vector{Cint}; kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    m, n = size(J)
    GC.@preserve devices begin
        check(ccall((:fdb_group_create_dense, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, ld(J), opts))
    end
    Group(h[], length(devices), nothing)
end

# fs[i]: the closure member i calls (its arrays live on devices[i]); x, jvals, fx, f_in live on devices[1]
function group_jacobian!(g::Group, jvals::CuArray{Float64}, fs::Vector, x::CuVector{Float64}, m::Integer;
        fx = nothing, f_in = nothing, relstep = nothing, absstep = relstep, dir = true)
    states = [FnState(f, m, length(x), nothing) for f in fs]
    ctxs = Ptr{Cvoid}[pointer_from_objref(s) for s in states]
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve states ctxs x jvals fx f_in begin
        rc = ccall((:fdb_group_jacobian, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64},
                Float64, Float64, Float64, Ptr{Cvoid}),
            g.handle, cf, pointer(ctxs), pointer(x), pointer(jvals), fx === nothing ? CU_NULL : pointer(fx),
            f_in === nothing ? CU_NULL : pointer(f_in), stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
    end
    for s in states
        s.err === nothing || throw(s.err)
    end
    check(rc)
    nothing
end

# ---- finite_difference_hessian! on several GPUs from ONE call: the i-blocks are split over `devices` (point-balanced,
#      contiguous ranges); devices[1] is the root and owns x, H and fx; every member evaluates f(x) and its own points and
#      stores its entries straight into the root's H, bit-identical to one device.  kw: max_batch, scratch_bytes, use_graph.
function group_hessian(H::CuMatrix{Float64}, n::Integer, devices::Vector{Cint}; kw...)
    size(H) == (n, n) || throw(DimensionMismatch("H must be $n x $n"))
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(FDB_HCENTRAL; kw...))
    GC.@preserve devices begin
        check(ccall((:fdb_group_create_hessian, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), n, ld(H), opts))
    end
    Group(h[], length(devices), nothing)
end

# fs[i]: the scalar f(x) member i calls (its arrays live on devices[i]); H, x and fx (a 1-element CuVector) live on devices[1]
function group_hessian!(g::Group, H::CuMatrix{Float64}, fs::Vector, x::CuVector{Float64};
        relstep = nothing, absstep = relstep, fx = nothing)
    states = [FnState(scalar_f(f), 1, length(x), nothing) for f in fs]
    ctxs = Ptr{Cvoid}[pointer_from_objref(s) for s in states]
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve states ctxs x H fx begin
        rc = ccall((:fdb_group_hessian, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, Float64, Float64,
                Ptr{Cvoid}),
            g.handle, cf, pointer(ctxs), pointer(x), pointer(H), fx === nothing ? CU_NULL : pointer(fx), stepval(relstep),
            stepval(absstep), CUDA.stream().handle)
    end
    for s in states
        s.err === nothing || throw(s.err)
    end
    check(rc)
    H
end

# ---- finite_difference_gradient! on several GPUs from ONE call: the dense group with m = 1 (df is J, 1 x n, ldJ = 1).
#      Member i owns a contiguous block of the n components (every component costs the same f calls) and writes its
#      entries of df straight into the root's df; devices[1] is the root and owns x and df.  Bit-identical to one device.
#      kw: max_batch, scratch_bytes, use_graph.  :complex groups are refused by fdb_group_jacobian (FDB_ERR_UNSUPPORTED).
mutable struct GradientGroup
    group::Group
    n::Int
    fdtype::Any
end

function group_gradient(n::Integer, devices::Vector{Cint}; fdtype = Val(:central), kw...)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    GC.@preserve devices begin
        check(ccall((:fdb_group_create_dense, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), 1, n, 1, opts))
    end
    GradientGroup(Group(h[], length(devices), nothing), n, fdtype)
end

# fs[i]: the scalar f(x) member i calls (its arrays live on devices[i]); df and x live on devices[1].  Forward mode: f(x)
# is evaluated once, by fs[1] at the root, unless fx (a Number or a 1-element CuVector, gradients.jl:409-410) is given,
# and passed to every member as f_in, so a call makes 1 + n evaluations (n with fx), as the reference does.
function group_gradient!(g::GradientGroup, df::CuVector{Float64}, fs::Vector, x::CuVector{Float64};
        fx = nothing, relstep = nothing, absstep = relstep, dir = true)
    length(x) == g.n || throw(DimensionMismatch("length(x) = $(length(x)), the group was built for $(g.n)"))
    length(df) == g.n || throw(DimensionMismatch("length(df) != length(x)"))
    length(fs) == g.group.n || throw(ArgumentError("one f per member"))
    f_in = nothing
    if fdcode(g.fdtype) == FDB_FORWARD
        if fx isa CuVector{Float64}
            length(fx) == 1 || throw(DimensionMismatch("fx must hold one value"))
            f_in = fx
        elseif fx !== nothing
            f_in = CuArray(Float64[fx])
        else
            f_in = CuVector{Float64}(undef, 1)
            scalar_f(fs[1])(f_in, x)
        end
    end
    states = [FnState(scalar_f(f), 1, g.n, nothing) for f in fs]
    ctxs = Ptr{Cvoid}[pointer_from_objref(s) for s in states]
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve states ctxs x df f_in begin
        rc = ccall((:fdb_group_jacobian, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64},
                Float64, Float64, Float64, Ptr{Cvoid}),
            g.group.handle, cf, pointer(ctxs), pointer(x), pointer(df), CU_NULL,
            f_in === nothing ? CU_NULL : pointer(f_in), stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
    end
    for s in states
        s.err === nothing || throw(s.err)
    end
    check(rc)
    df
end

# ---- column-block shards (few-colour problems on several GPUs): one process per GPU, each owning the columns c0+1:c1.
# `sub` is the block's pattern (colptr slice rebased to 1, rows rebased to the block's first row), `f_rows!` computes
# that row range from the x slice the rows depend on, `eps` holds the step sizes of the FULL x (color_eps! below).
function color_eps!(eps::CuVector{Float64}, epsplan::Plan, x::CuVector{Float64}; relstep = nothing, absstep = relstep, dir = true)
    check(ccall((:fdb_color_eps, libfdjac), Cint,
        (Ptr{Cvoid}, CuPtr{Float64}, Float64, Float64, Float64, CuPtr{Float64}, Ptr{Cvoid}),
        epsplan.handle, pointer(x), stepval(relstep), stepval(absstep), Float64(dir), pointer(eps), CUDA.stream().handle))
    eps
end

function eps_plan(n::Integer, colorvec::Vector{Int64}, fd::Cint)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fd))
    GC.@preserve colorvec begin
        check(ccall((:fdb_eps_plan_create, libfdjac), Cint, (Ref{Ptr{Cvoid}}, Int64, Ptr{Int64}, Ref{PlanOpts}),
            h, n, pointer(colorvec), opts))
    end
    Plan(h[], colorvec)
end

set_external_eps!(plan::Plan, eps::CuVector{Float64}) =
    check(ccall((:fdb_plan_set_external_eps, libfdjac), Cint, (Ptr{Cvoid}, CuPtr{Float64}), plan.handle, pointer(eps)))

# ---- out-of-place forms: J = finite_difference_jacobian(f, x, cache, f_in; …)  src/jacobians.jl:240-429, and
#      jvp = finite_difference_jvp(f, x, v, cache, f_in; …)  src/jvp.jl:133-189.  f(x) returns a new array; the trampoline
#      copies it into the slot the library hands out.
oop_f(f) = (fx, xv) -> (copyto!(fx, vec(f(xv))); nothing)

# mirror of fdb_oop_out (include/fdjac_b200.h)
struct OopOut
    J::CuPtr{Float64}
    colptr::CuPtr{Int64}
    rowval::CuPtr{Int64}
    nzval::CuPtr{Float64}
    cap::Int64
    nnz::CuPtr{Int64}
end

function oop_plan(anchor, sp, m::Integer, n::Integer, kind::Cint, ncols::Integer, colorvec, fd::Cint)
    key = (:oop, kind, m, n, ncols, sp === nothing ? 0 : objectid(sp.rowval), color_key(colorvec), fd)
    cached_plan(anchor, key) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve sp croot begin
            if sp === nothing
                check(ccall((:fdb_oop_plan_create_dense, libfdjac), Cint,
                    (Ref{Ptr{Cvoid}}, Int64, Int64, Ptr{Int64}, Int64, Cint, Int64, Ref{PlanOpts}),
                    h, m, n, cptr, ncols, kind, max(m, 1), opts))
            else
                check(ccall((:fdb_oop_plan_create_csc, libfdjac), Cint,
                    (Ref{Ptr{Cvoid}}, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
                    h, m, n, pointer(sp.colptr), pointer(sp.rowval), cptr, kind, max(m, 1), opts))
            end
        end
        Plan(h[], (sp, croot))
    end
end

hostcsc(A::DeviceCSC) = A.host
hostcsc(A::SparseMatrixCSC) = A
hostcsc(A) = throw(ArgumentError("not built: $(typeof(A)) in the out-of-place Jacobian (SparseMatrixCSC, DeviceCSC, a band " *
                                 "type or nothing)"))

# band sparsities the out-of-place Jacobian takes in closed form (fdb_oop_plan_create_banded): (m, n, l, u), else nothing.
# Their structural entries are the in-matrix band; Tridiagonal is the band (1, 1).
oopband(A::DeviceBanded) = A.l >= 0 && A.u >= 0 ? (A.m, A.n, A.l, A.u) : nothing
oopband(A::Union{DeviceDiagonal, DeviceBidiagonal, Diagonal, Bidiagonal, SymTridiagonal}) = (size(A, 1), size(A, 2), bands(A)...)
oopband(A::Union{Tridiagonal, DeviceTridiagonal}) = (size(A, 1), size(A, 2), 1, 1)
oopband(A) = nothing

function oop_band_plan(anchor, band, kind::Cint, colorvec, fd::Cint)
    m, n, l, u = band
    cached_plan(anchor, (:oop_band, kind, band, color_key(colorvec), fd)) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve croot begin
            check(ccall((:fdb_oop_plan_create_banded, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, Int64, Int64, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
                h, m, n, l, u, cptr, kind, max(m, 1), opts))
        end
        Plan(h[], croot)
    end
end

# block sparsities the out-of-place Jacobian takes in closed form (fdb_oop_plan_create_block_banded / _block_dense): their
# structural entries are those the in-place block plans write.  Only the sparse result is built.
oopblock(A::Union{DeviceBlockBanded, DeviceBlockDense}) = A
oopblock(A) = nothing

function oop_block_plan(anchor, B::DeviceBlockBanded, kind::Cint, colorvec, fd::Cint)
    cached_plan(anchor, (:oop_block_banded, kind, B.blocks, B.l, B.u, B.lam, B.mu, color_key(colorvec), fd)) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd))
        cptr, croot = color_arg(colorvec, sum(B.blocks))
        GC.@preserve croot B begin
            check(ccall((:fdb_oop_plan_create_block_banded, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Ptr{Int64}, Int64, Int64, Int64, Int64, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
                h, length(B.blocks), pointer(B.blocks), B.l, B.u, B.lam, B.mu, cptr, kind, max(sum(B.blocks), 1), opts))
        end
        Plan(h[], croot)
    end
end

function oop_block_plan(anchor, B::DeviceBlockDense, kind::Cint, colorvec, fd::Cint)
    cached_plan(anchor, (:oop_block_dense, kind, B.blocks, B.l, B.u, color_key(colorvec), fd)) do
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd))
        cptr, croot = color_arg(colorvec, sum(B.blocks))
        GC.@preserve croot B begin
            check(ccall((:fdb_oop_plan_create_block_dense, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Ptr{Int64}, Int64, Int64, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
                h, length(B.blocks), pointer(B.blocks), B.l, B.u, cptr, kind, max(sum(B.blocks), 1), opts))
        end
        Plan(h[], croot)
    end
end

# CSR results (fdb_oop_plan_create_csr): a DeviceCSR prototype with a DeviceCSR sparsity, or with a CSC one whose entry set
# is converted to CSR.  oopcsr gives the pattern the plan is made from (the DeviceCSR, or the host SparseMatrixCSC), else
# nothing; every other pairing with a DeviceCSR on either side throws ArgumentError, and a prototype of another size
# DimensionMismatch (the mirror's ValueError).
function oopcsr(sparsity, jac_prototype)
    sparsity isa DeviceCSR || jac_prototype isa DeviceCSR || return nothing
    jac_prototype isa DeviceCSR && sparsity isa Union{DeviceCSR, SparseMatrixCSC, DeviceCSC} ||
        throw(ArgumentError("not built: a $(typeof(sparsity)) sparsity with a $(typeof(jac_prototype)) jac_prototype " *
                            "(a DeviceCSR result takes a DeviceCSR, DeviceCSC or SparseMatrixCSC sparsity)"))
    size(jac_prototype) == size(sparsity) ||
        throw(DimensionMismatch("jac_prototype is $(size(jac_prototype)) but sparsity is $(size(sparsity))"))
    sparsity isa DeviceCSR ? sparsity : hostcsc(sparsity)
end

# the arrays that identify a CSR result's pattern (the plan cache's anchor and key), and the CSR arrays the plan takes:
# a DeviceCSR's own, or the CSR of a CSC's entry set (copy(transpose(A)): O(nnz), every stored entry kept, columns
# ascending in a row), built only when a plan is made
csrid(A::DeviceCSR) = (A.rowptr, A.colval)
csrid(A::SparseMatrixCSC) = (A.colptr, A.rowval)
csrarrays(A::DeviceCSR) = (A.rowptr, A.colval)
function csrarrays(A::SparseMatrixCSC)
    T = copy(transpose(A))
    (CuVector{Int64}(T.colptr), CuVector{Int64}(T.rowval))
end

function oop_csr_plan(src, m::Integer, n::Integer, colorvec, fd::Cint)
    anchor, second = csrid(src)
    cached_plan(anchor, (:oop_csr, m, n, objectid(second), color_key(colorvec), fd)) do
        rowptr, colval = csrarrays(src)
        h = Ref{Ptr{Cvoid}}(C_NULL)
        opts = Ref(PlanOpts(fd))
        cptr, croot = color_arg(colorvec, n)
        GC.@preserve croot rowptr colval begin
            check(ccall((:fdb_oop_plan_create_csr, libfdjac), Cint,
                (Ref{Ptr{Cvoid}}, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
                h, m, n, pointer(rowptr), pointer(colval), cptr, FDB_OOP_SPARSE, max(m, 1), opts))
        end
        Plan(h[], (rowptr, colval, croot))
    end
end

"""
    finite_difference_jacobian(f, x::CuVector{Float64}, cache::JacobianCache, f_in = nothing;
                               relstep, absstep, colorvec, sparsity, jac_prototype, dir)

`src/jacobians.jl:277-429` on the device.  The result follows (sparsity, jac_prototype) as `J + Ji` does in the reference:
a dense `CuMatrix` (raw quotients without either, `0.0 + dx` with a dense prototype or a CSC sparsity) or, with a sparse
prototype, a `DeviceCSC` holding the entries whose value is not ±0.0 (its pattern is copied back to the host: reading the
kept count is the call's one synchronisation).  A `DeviceBlockBanded` or `DeviceBlockDense` sparsity takes a sparse
prototype only (a dense result of it throws `ArgumentError`).  A `DeviceCSR` prototype with a `DeviceCSR`, `DeviceCSC` or
`SparseMatrixCSC` sparsity gives a `DeviceCSR` of the kept entries, rows in order and each row in the sparsity's storage
order (fdb_oop_plan_create_csr; a CSC sparsity is converted on the host).  `cache.x1` receives a copy of x (:293-295).
"""
function finite_difference_jacobian(f, x::CuVector{Float64},
        cache::JacobianCache{T1, T2, T3, T4, cType, sType, fdtype, returntype}, f_in = nothing;
        relstep = nothing, absstep = relstep, colorvec = cache.colorvec, sparsity = cache.sparsity,
        jac_prototype = nothing, dir = true) where {T1, T2, T3, T4, cType, sType, fdtype, returntype}
    cache.x1 === x || copyto!(cache.x1, x)
    n = length(x)
    csr = oopcsr(sparsity, jac_prototype)
    band = sparsity === nothing || csr !== nothing ? nothing : oopband(sparsity)
    block = sparsity === nothing || csr !== nothing ? nothing : oopblock(sparsity)
    sp = sparsity === nothing || band !== nothing || block !== nothing || csr !== nothing ? nothing : hostcsc(sparsity)
    m = csr !== nothing ? size(sparsity, 1) : band !== nothing ? band[1] : block !== nothing ? size(block, 1) :
        sp !== nothing ? size(sp, 1) : (f_in !== nothing ? length(f_in) : length(cache.fx))
    block !== nothing && !(jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC) &&
        throw(ArgumentError("not built: a dense out-of-place result of a $(typeof(block)) sparsity (give a sparse " *
                            "jac_prototype, or a CSC sparsity)"))
    if csr !== nothing
        kind, ncols = FDB_OOP_SPARSE, n
    elseif jac_prototype === nothing
        kind, ncols = sp === nothing && band === nothing ? (FDB_OOP_RAW, 0) : (FDB_OOP_DENSE, n)
    elseif jac_prototype isa AbstractMatrix && !(jac_prototype isa SparseMatrixCSC)
        kind, ncols = FDB_OOP_DENSE, size(jac_prototype, 2)
    else
        kind, ncols = FDB_OOP_SPARSE, size(hostcsc(jac_prototype), 2)
    end
    fd = fdcode(fdtype)
    plan = csr !== nothing ? oop_csr_plan(csr, m, n, colorvec, fd) :
           band !== nothing ? oop_band_plan(cache, band, kind, colorvec, fd) :
           block !== nothing ? oop_block_plan(cache, block, kind, colorvec, fd) :
           oop_plan(sp === nothing ? cache : sp.colptr, sp, m, n, kind, ncols, colorvec, fd)
    pinfo = info(plan)
    kind == FDB_OOP_RAW && (ncols = pinfo.n_local_colors)
    st = FnState(oop_f(f), m, n, nothing)
    J = nothing
    colptr = rowval = nzval = nnz = nothing
    if kind == FDB_OOP_SPARSE
        cap = sp === nothing && band === nothing && block === nothing && csr === nothing ? m * pinfo.n_local_colors :
              pinfo.n_entries
        # a CSR result: colptr receives the m + 1 row starts and rowval the columns
        colptr, rowval = CuVector{Int64}(undef, (csr === nothing ? ncols : m) + 1), CuVector{Int64}(undef, max(cap, 1))
        nzval, nnz = CuVector{Float64}(undef, max(cap, 1)), CuVector{Int64}(undef, 1)
        out = Ref(OopOut(CU_NULL, pointer(colptr), pointer(rowval), pointer(nzval), cap, pointer(nnz)))
    else
        J = CuMatrix{Float64}(undef, max(m, 1), ncols)
        out = Ref(OopOut(pointer(J), CU_NULL, CU_NULL, CU_NULL, 0, CU_NULL))
    end
    rc = Cint(0)
    GC.@preserve st x J colptr rowval nzval nnz f_in begin
        if fdtype == Val(:complex)
            cfc = @cfunction(f_trampoline_c, Cint, (Ptr{Cvoid}, CuPtr{ComplexF64}, CuPtr{ComplexF64}, Int64, Int64, Int64, Ptr{Cvoid}))
            rc = ccall((:fdb_jacobian_oop_complex, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, Ref{OopOut}, Ptr{Cvoid}),
                plan.handle, cfc, pointer_from_objref(st), pointer(x), out, CUDA.stream().handle)
        else
            cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
            rc = ccall((:fdb_jacobian_oop, libfdjac), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, Ref{OopOut}, CuPtr{Float64}, CuPtr{Float64},
                    Float64, Float64, Float64, Ptr{Cvoid}),
                plan.handle, cf, pointer_from_objref(st), pointer(x), out, CU_NULL,
                (f_in === nothing || fdtype != Val(:forward)) ? CU_NULL : pointer(f_in),
                stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
        end
    end
    st.err === nothing || throw(st.err)
    check(rc)
    kind == FDB_OOP_SPARSE || return m == 0 ? J[1:0, :] : J
    k = Int(Array(nnz)[1])                                     # the one host synchronisation
    csr === nothing || return DeviceCSR(m, n, colptr, rowval[1:k], nzval[1:k])
    host = SparseMatrixCSC(m, ncols, Array(colptr), Array(rowval[1:k]), zeros(k))
    DeviceCSC(host, nzval[1:k])
end

# ---- the out-of-place Jacobian on several GPUs from ONE call: the colours (dense branch: column blocks of the
#      maximum(colorvec) quotient columns) are split over `devices`; devices[1] is the root and owns x and the result, every
#      member writes exactly its own slots of it, and the root compacts a sparse result once every member has finished.
#      Bit-identical to finite_difference_jacobian on one device.  kw: max_batch, scratch_bytes, partition, use_graph.
mutable struct OopGroup
    group::Group
    kind::Cint
    m::Int
    n::Int
    ncols::Int         # columns of the result (the prototype's, else maximum(colorvec))
    cap::Int           # candidate entries of a sparse result
    fdtype::Any
    csr::Bool          # a DeviceCSR result (group_oop_csr): the pointer holds the m + 1 row starts
end

function oop_group_result(h, devices, roots, kind, m, n, ncols, fdtype)
    g = Group(h[], length(devices), roots)
    p0, pl = Ref{Ptr{Cvoid}}(C_NULL), Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:fdb_group_plan, libfdjac), Cint, (Ptr{Cvoid}, Cint, Ref{Ptr{Cvoid}}), g.handle, 0, p0))
    check(ccall((:fdb_group_plan, libfdjac), Cint, (Ptr{Cvoid}, Cint, Ref{Ptr{Cvoid}}), g.handle, length(devices) - 1, pl))
    i0 = Ref{PlanInfo}()
    check(ccall((:fdb_plan_info, libfdjac), Cint, (Ptr{Cvoid}, Ref{PlanInfo}), p0[], i0))
    b, e = Ref{Int64}(0), Ref{Int64}(0)
    check(ccall((:fdb_plan_dense_range, libfdjac), Cint, (Ptr{Cvoid}, Ref{Int64}, Ref{Int64}), pl[], b, e))
    kind == FDB_OOP_RAW && (ncols = e[])                       # C of the whole result: where the last block ends
    OopGroup(g, kind, m, n, ncols, i0[].n_entries, fdtype, false)
end

# sparsity: a CSC pattern (SparseMatrixCSC or DeviceCSC); jac_prototype: nothing, a dense matrix or a sparse one
function group_oop_csc(sparsity, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    sp = hostcsc(sparsity)
    m, n = size(sp)
    kind = jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC ? FDB_OOP_SPARSE : FDB_OOP_DENSE
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve sp croot devices begin
        check(ccall((:fdb_group_create_oop_csc, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, pointer(sp.colptr), pointer(sp.rowval), cptr, kind, max(m, 1), opts))
    end
    oop_group_result(h, devices, (sp, croot), kind, m, n, n, fdtype)
end

# sparsity: a band type oopband takes (DeviceBanded with l, u >= 0, Diagonal, Bidiagonal, SymTridiagonal, Tridiagonal)
function group_oop_banded(sparsity, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    band = oopband(sparsity)
    band === nothing && throw(ArgumentError("not built: $(typeof(sparsity)) as a band sparsity"))
    m, n, l, u = band
    kind = jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC ? FDB_OOP_SPARSE : FDB_OOP_DENSE
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve croot devices begin
        check(ccall((:fdb_group_create_oop_banded, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Int64, Int64, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, l, u, cptr, kind, max(m, 1), opts))
    end
    oop_group_result(h, devices, croot, kind, m, n, n, fdtype)
end

# sparsity: a DeviceBlockBanded / DeviceBlockDense; jac_prototype: a sparse one (the dense result is not built)
function group_oop_block_banded(B::DeviceBlockBanded, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC ||
        throw(ArgumentError("not built: a dense out-of-place result of a block-banded sparsity"))
    n = sum(B.blocks)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve B croot devices begin
        check(ccall((:fdb_group_create_oop_block_banded, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Ptr{Int64}, Int64, Int64, Int64, Int64, Ptr{Int64}, Cint, Int64,
                Ref{PlanOpts}),
            h, length(devices), pointer(devices), length(B.blocks), pointer(B.blocks), B.l, B.u, B.lam, B.mu, cptr,
            FDB_OOP_SPARSE, max(n, 1), opts))
    end
    oop_group_result(h, devices, croot, FDB_OOP_SPARSE, n, n, n, fdtype)
end

function group_oop_block_dense(B::DeviceBlockDense, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC ||
        throw(ArgumentError("not built: a dense out-of-place result of a block-dense sparsity"))
    n = sum(B.blocks)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve B croot devices begin
        check(ccall((:fdb_group_create_oop_block_dense, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Ptr{Int64}, Int64, Int64, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), length(B.blocks), pointer(B.blocks), B.l, B.u, cptr, FDB_OOP_SPARSE,
            max(n, 1), opts))
    end
    oop_group_result(h, devices, croot, FDB_OOP_SPARSE, n, n, n, fdtype)
end

# sparsity: a DeviceCSR, or a CSC pattern (converted on the host); jac_prototype: a DeviceCSR of the same size
function group_oop_csr(sparsity, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    rowptr, colval = csrarrays(oopcsr(sparsity, jac_prototype))
    m, n = size(sparsity)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve rowptr colval croot devices begin
        check(ccall((:fdb_group_create_oop_csr, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Ptr{Int64}, Cint, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, pointer(rowptr), pointer(colval), cptr, FDB_OOP_SPARSE, max(m, 1), opts))
    end
    g = oop_group_result(h, devices, (rowptr, colval, croot), FDB_OOP_SPARSE, m, n, n, fdtype)
    g.csr = true
    g
end

# sparsity === nothing: m rows (length of f(x)), n = length(x)
function group_oop_dense(m::Integer, n::Integer, colorvec, fdtype, devices::Vector{Cint}; jac_prototype = nothing, kw...)
    if jac_prototype === nothing
        kind, ncols = FDB_OOP_RAW, 0
    elseif jac_prototype isa SparseMatrixCSC || jac_prototype isa DeviceCSC
        kind, ncols = FDB_OOP_SPARSE, size(hostcsc(jac_prototype), 2)
    else
        kind, ncols = FDB_OOP_DENSE, size(jac_prototype, 2)
    end
    h = Ref{Ptr{Cvoid}}(C_NULL)
    opts = Ref(PlanOpts(fdcode(fdtype); kw...))
    cptr, croot = color_arg(colorvec, n)
    GC.@preserve croot devices begin
        check(ccall((:fdb_group_create_oop_dense, libfdjac), Cint,
            (Ref{Ptr{Cvoid}}, Cint, Ptr{Cint}, Int64, Int64, Ptr{Int64}, Int64, Cint, Int64, Ref{PlanOpts}),
            h, length(devices), pointer(devices), m, n, cptr, ncols, kind, max(m, 1), opts))
    end
    oop_group_result(h, devices, croot, kind, m, n, ncols, fdtype)
end

# fs[i]: the out-of-place f(x) member i calls (its arrays live on devices[i]); x and f_in live on devices[1].  In forward mode
# without f_in, f(x) is evaluated once by fs[1] at the root and passed on as f_in (:299-300): 1 + C calls in all.
function group_jacobian(g::OopGroup, fs::Vector, x::CuVector{Float64}; f_in = nothing, relstep = nothing,
        absstep = relstep, dir = true)
    length(x) == g.n || throw(DimensionMismatch("length(x) = $(length(x)), the group was built for $(g.n)"))
    fd = fdcode(g.fdtype)
    if f_in === nothing && fd == FDB_FORWARD
        f_in = vec(fs[1](x))
    end
    f_in === nothing || length(f_in) == g.m || throw(DimensionMismatch("length(f_in) != $(g.m)"))
    states = [FnState(oop_f(f), g.m, g.n, nothing) for f in fs]
    ctxs = Ptr{Cvoid}[pointer_from_objref(s) for s in states]
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    J = nothing
    colptr = rowval = nzval = nnz = nothing
    if g.kind == FDB_OOP_SPARSE
        colptr, rowval = CuVector{Int64}(undef, (g.csr ? g.m : g.ncols) + 1), CuVector{Int64}(undef, max(g.cap, 1))
        nzval, nnz = CuVector{Float64}(undef, max(g.cap, 1)), CuVector{Int64}(undef, 1)
        out = Ref(OopOut(CU_NULL, pointer(colptr), pointer(rowval), pointer(nzval), g.cap, pointer(nnz)))
    else
        J = CuMatrix{Float64}(undef, max(g.m, 1), g.ncols)
        out = Ref(OopOut(pointer(J), CU_NULL, CU_NULL, CU_NULL, 0, CU_NULL))
    end
    rc = Cint(0)
    GC.@preserve states ctxs x J colptr rowval nzval nnz f_in begin
        rc = ccall((:fdb_group_jacobian_oop, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}, CuPtr{Float64}, Ref{OopOut}, CuPtr{Float64}, CuPtr{Float64},
                Float64, Float64, Float64, Ptr{Cvoid}),
            g.group.handle, cf, pointer(ctxs), pointer(x), out, CU_NULL,
            (f_in === nothing || fd != FDB_FORWARD) ? CU_NULL : pointer(f_in),
            stepval(relstep), stepval(absstep), Float64(dir), CUDA.stream().handle)
    end
    for s in states
        s.err === nothing || throw(s.err)
    end
    check(rc)
    g.kind == FDB_OOP_SPARSE || return g.m == 0 ? J[1:0, :] : J
    k = Int(Array(nnz)[1])                                     # the one host synchronisation
    g.csr && return DeviceCSR(g.m, g.n, colptr, rowval[1:k], nzval[1:k])
    host = SparseMatrixCSC(g.m, g.ncols, Array(colptr), Array(rowval[1:k]), zeros(k))
    DeviceCSC(host, nzval[1:k])
end

# cache-less form :240-259: f(x) once, then the cached form with it as f_in
function finite_difference_jacobian(f, x::CuVector{Float64}, fdtype = Val(:forward), returntype = eltype(x), f_in = nothing;
        kw...)
    fdtype isa Type && (fdtype = fdtype())
    fx = f_in === nothing ? f(x) : f_in
    cache = JacobianCache(x, fdtype == Val(:complex) ? real(fx) : fx, fdtype, returntype)
    finite_difference_jacobian(f, x, cache, fdtype == Val(:complex) ? real(fx) : fx; kw...)
end

"""
    finite_difference_jvp(f, x::CuVector{Float64}, v::CuVector{Float64}, cache::JVPCache, f_in = nothing; relstep, absstep, dir)

`src/jvp.jl:159-189` on the device (fdb_jvp_oop): central mode evaluates f(x + εv) before f(x − εv).  Returns a new
`CuVector{Float64}`; the cache arrays are not written.
"""
function finite_difference_jvp(f, x::CuVector{Float64}, v::CuVector{Float64}, cache::JVPCache{X1, FX1, fdtype},
        f_in = nothing; relstep = nothing, absstep = relstep, dir = true) where {X1, FX1, fdtype}
    fdtype == Val(:complex) && error("finite_difference_jvp doesn't support :complex-mode finite diff")
    m, n = f_in === nothing ? length(cache.fx1) : length(f_in), length(x)
    plan = jvp_plan(m, n, fdcode(fdtype))
    jvp, x1, fx1 = CuVector{Float64}(undef, m), CuVector{Float64}(undef, n), CuVector{Float64}(undef, m)
    st = FnState(oop_f(f), m, n, nothing)
    cf = @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid}))
    rc = Cint(0)
    GC.@preserve st jvp x v x1 fx1 f_in begin
        rc = ccall((:fdb_jvp_oop, libfdjac), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64}, CuPtr{Float64},
                CuPtr{Float64}, Float64, Float64, Float64, Ptr{Cvoid}),
            plan.handle, cf, pointer_from_objref(st), pointer(jvp), pointer(x), pointer(v), pointer(x1), pointer(fx1),
            (f_in === nothing || fdtype != Val(:forward)) ? CU_NULL : pointer(f_in), stepval(relstep), stepval(absstep),
            Float64(dir), CUDA.stream().handle)
    end
    st.err === nothing || throw(st.err)
    check(rc)
    jvp
end

# cache-less form :133-146
function finite_difference_jvp(f, x::CuVector{Float64}, v::CuVector{Float64}, fdtype = Val(:forward), f_in = nothing;
        kw...)
    fdtype isa Type && (fdtype = fdtype())
    fx = f_in === nothing ? f(x) : f_in
    finite_difference_jvp(f, x, v, JVPCache(x, fx, fdtype), fx; kw...)
end

end # module
