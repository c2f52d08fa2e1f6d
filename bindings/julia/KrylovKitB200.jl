# KrylovKitB200.jl — the reference-side binding of libb200krylov.so (include/b200krylov.h).
#
# STATUS: written against KrylovKit.jl v0.10.4 / VectorInterface.jl 0.5 signatures, NOT RUN: there is no
# Julia in the build image.  The Python package krylovkit.jl_b200/ binds the same C-ABI entry points in
# the same pairing and is what the test-suite exercises (INTEGRATION.md §6).  Everything below is a
# one-to-one `ccall`; no numerical code lives here.
#
# Usage:
#     using KrylovKit, KrylovKitB200
#     ctx = B200Ctx(size(A, 1), 40)                  # n rows, 40 slab columns (≈ krylovdim + 10)
#     op  = B200CSR(ctx, A)                          # A::SparseMatrixCSC{Float64,Int64}
#     x0  = B200Vec(ctx, rand(size(A, 1)))
#     vals, vecs, info = eigsolve(op, x0, 4, :SR, Lanczos(; orth = ClassicalGramSchmidt2()))
module KrylovKitB200

using KrylovKit, VectorInterface, LinearAlgebra, SparseArrays
import KrylovKit: OrthonormalBasis, Orthogonalizer, apply, apply_normal, apply_adjoint
import KrylovKit: project!!, unproject!!, rank1update!, basistransform!, orthogonalize!!
import KrylovKit: LanczosIterator, LanczosFactorization, expand!, normres
import KrylovKit: ClassicalGramSchmidt, ModifiedGramSchmidt, ClassicalGramSchmidt2, ModifiedGramSchmidt2,
    ClassicalGramSchmidtIR, ModifiedGramSchmidtIR

export B200Ctx, B200Vec, B200CSR, B200Dense

const lib = get(ENV, "B200KRYLOV_LIB", "libb200krylov.so")

# ---- status codes -> exceptions (include/b200krylov.h: B2K_OK … B2K_ENOTSUP) -------------------------
function check(ctxh::Ptr{Cvoid}, st::Cint)
    st == 0 && return nothing
    msg = unsafe_string(ccall((:b2k_last_error, lib), Cstring, (Ptr{Cvoid},), ctxh))
    st == -1 && throw(ArgumentError(msg))            # B2K_EINVAL
    st == -2 && throw(DimensionMismatch(msg))        # B2K_EDIM   (orthonormal.jl:93,140,158-161)
    error("b200krylov [$st]: $msg")                   # CUDA / memory / NCCL / not supported
end

# ---- context -------------------------------------------------------------------------------------------
mutable struct B200Ctx
    h::Ptr{Cvoid}          # C_NULL once destroyed: Julia runs finalizers in no particular order, so a vector's
    n::Int                 # finalizer may run AFTER its context's — every call below checks `alive(ctx)` first
    T::DataType
    spaces::Vector{Int}    # length of the vectors of each space (space 0 = n)
end
alive(ctx::B200Ctx) = ctx.h != C_NULL
function destroy!(ctx::B200Ctx)
    if alive(ctx)
        ccall((:b2k_ctx_destroy, lib), Cint, (Ptr{Cvoid},), ctx.h)
        ctx.h = C_NULL      # vectors / operators that outlive the context become inert instead of dangling
    end
    return nothing
end
function B200Ctx(n::Integer, ncols::Integer; T::Type{<:Union{Float64, Float32}} = Float64, device::Integer = 0)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(C_NULL, ccall((:b2k_ctx_create, lib), Cint, (Ref{Ptr{Cvoid}}, Cint, Int64, Cint, Cint),
                        h, device, n, ncols, T === Float64 ? 0 : 1))
    ctx = B200Ctx(h[], n, T, [Int(n)])
    finalizer(destroy!, ctx)
    return ctx
end
# one process per GPU: uid = 128 bytes from b2k_nccl_unique_id on rank 0, broadcast by MPI / Distributed
function B200Ctx(nlocal::Integer, ncols::Integer, rank::Integer, nranks::Integer, uid::Vector{UInt8},
                 nglobal::Integer, rowoffset::Integer; T = Float64, device::Integer = 0)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(C_NULL, ccall((:b2k_ctx_create_dist, lib), Cint,
                        (Ref{Ptr{Cvoid}}, Cint, Int64, Cint, Cint, Cint, Cint, Ptr{UInt8}, Int64, Int64),
                        h, device, nlocal, ncols, T === Float64 ? 0 : 1, rank, nranks, uid, nglobal, rowoffset))
    ctx = B200Ctx(h[], nlocal, T, [Int(nlocal)])
    finalizer(destroy!, ctx)
    return ctx
end
# additional vector space (the short side of GKL / LSMR): returns its index
function addspace!(ctx::B200Ctx, n::Integer, ncols::Integer; sharded::Bool = false)
    sp = Ref{Cint}(0)
    check(ctx.h, ccall((:b2k_space_create, lib), Cint, (Ptr{Cvoid}, Int64, Cint, Cint, Ref{Cint}),
                       ctx.h, n, ncols, sharded ? 1 : 0, sp))
    push!(ctx.spaces, Int(n))
    return Int(sp[])
end

# ---- vectors: one slab column each ----------------------------------------------------------------------
mutable struct B200Vec{T}
    ctx::B200Ctx
    handle::Int32
end
function B200Vec(ctx::B200Ctx; space::Integer = 0)
    v = Ref{Int32}(0)
    check(ctx.h, ccall((:b2k_vec_alloc, lib), Cint, (Ptr{Cvoid}, Cint, Ref{Int32}), ctx.h, space, v))
    return adopt(ctx, v[])
end
# wrap a column the library allocated (b2k_lanczos_expand_many); the finalizer returns it to the slab — unless the
# context is already gone (then its slab is gone too) or the library took the column back (`disown!`)
function adopt(ctx::B200Ctx, handle::Integer)
    x = B200Vec{ctx.T}(ctx, Int32(handle))
    finalizer(x) do y
        if y.handle >= 0 && alive(y.ctx)
            ccall((:b2k_vec_free, lib), Cint, (Ptr{Cvoid}, Int32), y.ctx.h, y.handle)
        end
    end
    return x
end
disown!(x) = (x.handle = Int32(-1); x)
Base.length(x::B200Vec) = x.ctx.spaces[space(x) + 1]
function B200Vec(ctx::B200Ctx, host::Vector{T}; space::Integer = 0) where {T}
    T === ctx.T || throw(ArgumentError("host data must be $(ctx.T)"))
    length(host) == ctx.spaces[space + 1] ||
        throw(DimensionMismatch("host vector has $(length(host)) entries, space $space holds $(ctx.spaces[space + 1])"))
    x = B200Vec(ctx; space = space)
    check(ctx.h, ccall((:b2k_vec_upload, lib), Cint, (Ptr{Cvoid}, Int32, Ptr{T}), ctx.h, x.handle, host))
    return x
end
function Base.Array(x::B200Vec{T}) where {T}
    out = Vector{T}(undef, length(x))
    check(x.ctx.h, ccall((:b2k_vec_download, lib), Cint, (Ptr{Cvoid}, Int32, Ptr{T}), x.ctx.h, x.handle, out))
    return out
end
space(x::B200Vec) = Int(x.handle >> 20)
_copy(x::B200Vec) = (y = B200Vec(x.ctx; space = space(x));
    check(x.ctx.h, ccall((:b2k_vec_copy, lib), Cint, (Ptr{Cvoid}, Int32, Int32), x.ctx.h, y.handle, x.handle)); y)

# ---- VectorInterface: the complete list KrylovKit uses (src/innerproductvec.jl:82-137) ------------------
VectorInterface.scalartype(::Type{B200Vec{T}}) where {T} = T

function VectorInterface.zerovector(x::B200Vec, ::Type{S} = scalartype(x)) where {S <: Number}
    S === scalartype(x) || throw(ArgumentError("B200Vec is real $(scalartype(x)) only"))
    y = B200Vec(x.ctx; space = space(x))
    return zerovector!(y)
end
function VectorInterface.zerovector!(x::B200Vec)
    check(x.ctx.h, ccall((:b2k_vec_zero, lib), Cint, (Ptr{Cvoid}, Int32), x.ctx.h, x.handle))
    return x
end
VectorInterface.zerovector!!(x::B200Vec) = zerovector!(x)

function VectorInterface.scale!(y::B200Vec, x::B200Vec, α::Number)      # y ← α x   (lanczos.jl:257, arnoldi.jl:209)
    check(y.ctx.h, ccall((:b2k_vec_scale, lib), Cint, (Ptr{Cvoid}, Int32, Int32, Float64),
                         y.ctx.h, y.handle, x.handle, Float64(α)))
    return y
end
VectorInterface.scale!(x::B200Vec, α::Number) = scale!(x, x, α)
VectorInterface.scale!!(x::B200Vec, α::Number) = scale!(x, x, α)
VectorInterface.scale!!(y::B200Vec, x::B200Vec, α::Number) = scale!(y, x, α)
VectorInterface.scale(x::B200Vec, α::Number) = scale!(B200Vec(x.ctx; space = space(x)), x, α)

function VectorInterface.add!(y::B200Vec, x::B200Vec, α::Number = 1, β::Number = 1)   # y ← β y + α x
    check(y.ctx.h, ccall((:b2k_vec_axpby, lib), Cint, (Ptr{Cvoid}, Int32, Int32, Float64, Float64),
                         y.ctx.h, y.handle, x.handle, Float64(α), Float64(β)))
    return y
end
VectorInterface.add!!(y::B200Vec, x::B200Vec, α::Number = 1, β::Number = 1) = add!(y, x, α, β)
VectorInterface.add(y::B200Vec, x::B200Vec, α::Number = 1, β::Number = 1) = add!(_copy(y), x, α, β)

function VectorInterface.inner(x::B200Vec, y::B200Vec)
    o = Ref{Float64}(0)
    check(x.ctx.h, ccall((:b2k_vec_inner, lib), Cint, (Ptr{Cvoid}, Int32, Int32, Ref{Float64}),
                         x.ctx.h, x.handle, y.handle, o))
    return o[]
end
function LinearAlgebra.norm(x::B200Vec)
    o = Ref{Float64}(0)
    check(x.ctx.h, ccall((:b2k_vec_norm, lib), Cint, (Ptr{Cvoid}, Int32, Ref{Float64}), x.ctx.h, x.handle, o))
    return o[]
end

# ---- operators (src/apply.jl) -----------------------------------------------------------------------------
mutable struct B200CSR{T}
    ctx::B200Ctx
    h::Ptr{Cvoid}
    adj::Any                              # A' (a B200CSR), built on the device by the first apply_adjoint
end
B200CSR{T}(ctx::B200Ctx, h::Ptr{Cvoid}) where {T} = B200CSR{T}(ctx, h, nothing)
function B200CSR(ctx::B200Ctx, A::SparseMatrixCSC{T, Int64}) where {T}      # colptr / rowval / nzval as stored
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ctx.h, ccall((:b2k_op_create_csc, lib), Cint,
                       (Ptr{Cvoid}, Ref{Ptr{Cvoid}}, Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{T}, Cint, Cint),
                       ctx.h, h, size(A, 1), size(A, 2), nnz(A), A.colptr, A.rowval, A.nzval, 8, 1))
    return B200CSR{T}(ctx, h[])          # the context owns the operator's device memory
end
mutable struct B200Dense{T}
    ctx::B200Ctx
    h::Ptr{Cvoid}
    space_in::Int                         # x of y = A x lives here (length n); y in space 0 (length m)
end
function B200Dense(ctx::B200Ctx, A::Matrix{T}, space_in::Integer) where {T}
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ctx.h, ccall((:b2k_op_create_dense, lib), Cint, (Ptr{Cvoid}, Ref{Ptr{Cvoid}}, Int64, Int64, Ptr{T}, Int64),
                       ctx.h, h, size(A, 1), size(A, 2), A, stride(A, 2)))
    return B200Dense{T}(ctx, h[], space_in)
end

function apply(A::B200CSR, x::B200Vec)                                          # apply.jl:1 — a NEW vector
    y = B200Vec(x.ctx; space = space(x))
    check(x.ctx.h, ccall((:b2k_op_apply, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32), x.ctx.h, A.h, x.handle, y.handle))
    return y
end
function apply(A::B200CSR, x::B200Vec, α₀::Number, α₁::Number)                   # apply.jl:4-11
    y = B200Vec(x.ctx; space = space(x))
    check(x.ctx.h, ccall((:b2k_op_apply_shifted, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Float64, Float64),
                         x.ctx.h, A.h, x.handle, y.handle, Float64(α₀), Float64(α₁)))
    return y
end
function apply_normal(A::B200Dense, x::B200Vec)                                  # apply.jl:14
    y = B200Vec(x.ctx; space = 0)
    check(x.ctx.h, ccall((:b2k_op_apply, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32), x.ctx.h, A.h, x.handle, y.handle))
    return y
end
function apply_adjoint(A::B200Dense, x::B200Vec)                                 # apply.jl:15
    y = B200Vec(x.ctx; space = A.space_in)
    check(x.ctx.h, ccall((:b2k_op_apply_adjoint, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32), x.ctx.h, A.h, x.handle, y.handle))
    return y
end
apply(A::B200Dense, x::B200Vec) = apply_normal(A, x)
# A' of a CSR operator, assembled on the device from A's arrays (b2k_op_create_transpose): the CSR of A' with sorted
# columns, so products with it have the bits of a host-built transpose.  apply_adjoint builds it once per operator,
# which lets KrylovKit's own bieigsolve, svdsolve and lssolve take a B200CSR.
function Base.adjoint(A::B200CSR{T}) where {T}
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(A.ctx.h, ccall((:b2k_op_create_transpose, lib), Cint, (Ptr{Cvoid}, Ref{Ptr{Cvoid}}, Ptr{Cvoid}),
                         A.ctx.h, h, A.h))
    return B200CSR{T}(A.ctx, h[])
end
apply_normal(A::B200CSR, x::B200Vec) = apply(A, x)                               # apply.jl:14
function apply_adjoint(A::B200CSR, x::B200Vec)                                   # apply.jl:15
    A.adj === nothing && (A.adj = adjoint(A))
    return apply(A.adj, x)
end
# (A x, A'(A x)) from ONE pass over the dense A — the building block of the flagged one-pass GKL step (no KrylovKit
# counterpart: gkl.jl:308-323 calls apply_adjoint and apply_normal separately).  A gklrecurrence specialisation on
# `GKLIterator{<:B200Dense}` would keep G = A'U next to U and recover A'u_{k+1} = (z - G c) / beta with unproject!!,
# guarded by the error estimate described in krylovkit.jl_b200/factorizations/gkl.py.
function apply_normal_gram(A::B200Dense, x::B200Vec)
    y = B200Vec(x.ctx; space = 0)
    z = B200Vec(x.ctx; space = A.space_in)
    check(x.ctx.h, ccall((:b2k_op_apply_normal_gram, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32),
                         x.ctx.h, A.h, x.handle, y.handle, z.handle))
    return y, z
end

# ---- Block (BlockLanczos) — factorizations/blocklanczos.jl:10-52, 277-353 -----------------------------------
# The reference runs these as loops of single-vector calls (p applies, p*q inners, p*k MGS steps); here each is one
# library call: SpMM for apply(A, ::Block), one multi-right-hand-side launch for block_inner, the library's
# block_reorthogonalize! / block_qr! with the reference's arithmetic (rank drop below tol, DGKS drift pass).
import KrylovKit: Block, block_inner, block_reorthogonalize!, block_qr!
const B200Block = Block{<:B200Vec}
_handles(b::B200Block) = Int32[v.handle for v in b.vec]
_ctx(b::B200Block) = b.vec[1].ctx

function apply(A::B200CSR, X::B200Block)                                         # blocklanczos.jl:38
    Y = [B200Vec(x.ctx; space = space(x)) for x in X.vec]
    hy = Int32[y.handle for y in Y]
    check(_ctx(X).h, ccall((:b2k_op_apply_block, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int32}, Ptr{Int32}, Cint),
                           _ctx(X).h, A.h, _handles(X), hy, length(X)))
    return Block(Y)
end
function block_inner(B₁::B200Block, B₂::B200Block)                               # blocklanczos.jl:43-52
    M = Matrix{Float64}(undef, length(B₁), length(B₂))
    check(_ctx(B₁).h, ccall((:b2k_block_inner, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Ptr{Int32}, Cint, Ptr{Float64}),
                            _ctx(B₁).h, _handles(B₁), length(B₁), _handles(B₂), length(B₂), M))
    return M
end
function block_reorthogonalize!(R::B200Block, V::OrthonormalBasis{<:B200Vec})    # blocklanczos.jl:277-284
    hv = Int32[q.handle for q in V]
    check(_ctx(R).h, ccall((:b2k_block_reorthogonalize, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Ptr{Int32}, Cint),
                           _ctx(R).h, _handles(R), length(R), hv, length(hv)))
    return R
end
function block_qr!(block::B200Block, tol::Real)                                  # blocklanczos.jl:312-353
    p = length(block)
    R = zeros(Float64, p, p)
    good = zeros(Int32, p)
    drift = Ref{Int32}(0)
    check(_ctx(block).h, ccall((:b2k_block_qr, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Float64, Ptr{Float64}, Ptr{Int32}, Ref{Int32}),
                               _ctx(block).h, _handles(block), p, Float64(tol), R, good, drift))
    good_idx = findall(!=(0), good)
    return R[good_idx, :], good_idx, drift[] != 0
end

# ---- basis fast path: what `Array` gets via _use_multithreaded_array_kernel (orthonormal.jl:66-73) --------
const B200Basis = OrthonormalBasis{<:B200Vec}
_cols(b::B200Basis, r) = Int32[b[i].handle for i in r]
_ctx(b::B200Basis) = b[1].ctx

function project!!(y::AbstractVector, b::B200Basis, x::B200Vec, α::Number = true, β::Number = false,
                   r = Base.OneTo(length(b)))                                    # orthonormal.jl:88-118
    length(y) == length(r) || throw(DimensionMismatch())
    h = β == 0 ? Vector{Float64}(undef, length(r)) : Vector{Float64}(y)
    check(x.ctx.h, ccall((:b2k_basis_project, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Int32, Float64, Float64, Ptr{Float64}),
                         x.ctx.h, _cols(b, r), length(r), x.handle, Float64(α), Float64(β), h))
    y .= h
    return y
end
function unproject!!(y::B200Vec, b::B200Basis, x::AbstractVector, α::Number = true, β::Number = false,
                     r = Base.OneTo(length(b)))                                  # orthonormal.jl:132-196
    length(x) == length(r) || throw(DimensionMismatch())
    check(y.ctx.h, ccall((:b2k_basis_unproject, lib), Cint, (Ptr{Cvoid}, Int32, Ptr{Int32}, Cint, Ptr{Float64}, Float64, Float64),
                         y.ctx.h, y.handle, _cols(b, r), length(r), Vector{Float64}(x), Float64(α), Float64(β)))
    return y
end
function rank1update!(b::B200Basis, y::B200Vec, x::AbstractVector, α::Number = true, β::Number = true,
                      r = Base.OneTo(length(b)))                                 # orthonormal.jl:210-275
    check(y.ctx.h, ccall((:b2k_basis_rank1update, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Int32, Ptr{Float64}, Float64, Float64),
                         y.ctx.h, _cols(b, r), length(r), y.handle, Vector{Float64}(x), Float64(α), Float64(β)))
    return b
end
function basistransform!(b::B200Basis, U::AbstractMatrix)                         # orthonormal.jl:291-354, in place
    m, keep = size(U)
    m == length(b) || throw(DimensionMismatch())
    Ud = Matrix{Float64}(U)
    check(_ctx(b).h, ccall((:b2k_basis_transform, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Ptr{Float64}, Cint, Cint),
                           _ctx(b).h, _cols(b, 1:m), m, Ud, m, keep))
    return b
end

_tag(::ClassicalGramSchmidt) = (0, 0.0);   _tag(::ModifiedGramSchmidt) = (1, 0.0)
_tag(::ClassicalGramSchmidt2) = (2, 0.0);  _tag(::ModifiedGramSchmidt2) = (3, 0.0)
_tag(a::ClassicalGramSchmidtIR) = (4, Float64(a.η));  _tag(a::ModifiedGramSchmidtIR) = (5, Float64(a.η))

function orthogonalize!!(v::B200Vec, b::B200Basis, x::AbstractVector, alg::Orthogonalizer)   # orthonormal.jl:378-452
    k = length(b)
    tag, η = _tag(alg)
    h = Vector{Float64}(undef, k); nrm = Ref{Float64}(0); passes = Ref{Cint}(0)
    check(v.ctx.h, ccall((:b2k_basis_orthogonalize, lib), Cint,
                         (Ptr{Cvoid}, Int32, Ptr{Int32}, Cint, Ptr{Float64}, Cint, Float64, Ref{Float64}, Ref{Cint}),
                         v.ctx.h, v.handle, _cols(b, 1:k), k, h, tag, η, nrm, passes))
    x[1:k] .= h
    return (v, x)
end
function orthogonalize!!(v::B200Vec, q::B200Vec, alg::Orthogonalizer)             # orthonormal.jl:455-489
    tag, η = _tag(alg)
    s = Ref{Float64}(0); nrm = Ref{Float64}(0)
    check(v.ctx.h, ccall((:b2k_vec_orthogonalize, lib), Cint, (Ptr{Cvoid}, Int32, Int32, Cint, Float64, Ref{Float64}, Ref{Float64}),
                         v.ctx.h, v.handle, q.handle, tag, η, s, nrm))
    return (v, s[])
end

function LinearAlgebra.rmul!(b::B200Basis, G::LinearAlgebra.Givens)               # dense/givens.jl:12-36
    check(_ctx(b).h, ccall((:b2k_basis_givens, lib), Cint, (Ptr{Cvoid}, Int32, Int32, Float64, Float64),
                           _ctx(b).h, b[G.i1].handle, b[G.i2].handle, Float64(G.c), Float64(G.s)))
    return b
end
function LinearAlgebra.rmul!(b::B200Basis, H::KrylovKit.Householder)              # dense/reflector.jl:143-154
    work = B200Vec(_ctx(b); space = space(b[1]))
    check(_ctx(b).h, ccall((:b2k_basis_householder, lib), Cint, (Ptr{Cvoid}, Ptr{Int32}, Cint, Ptr{Float64}, Float64, Int32),
                           _ctx(b).h, _cols(b, H.r), length(H.r), Vector{Float64}(H.v), Float64(H.β), work.handle))
    return b
end

# ---- fused steps: the path bench.py times (DESIGN.md §3, §4) ---------------------------------------------------
# expand!(iter::LanczosIterator, state) — src/factorizations/lanczos.jl:250-272.  For a device CSR operator one
# C-ABI call does `V <- push!(V, r/β); w = A v; lanczosrecurrence` with ONE host synchronisation; with
# ClassicalGramSchmidt2 it is two launches (SpMV with the normalisation fused into its gather + one cooperative
# Gram-Schmidt kernel).  Same operation order as lanczos.jl:313-324, same α, β, V, r as the generic method.
function expand!(iter::LanczosIterator{<:B200CSR}, state::LanczosFactorization; verbosity::Int = KrylovKit.KrylovDefaults.verbosity[])
    expand_many!(iter, state, 1, zero(Float64))
    return state
end

# `nsteps` consecutive expand! calls — the `while K < krylovdim && β > tol` loop of src/eigsolve/lanczos.jl:45-79 —
# in one C-ABI call (b2k_lanczos_expand_many): with ClassicalGramSchmidt2 the steps are chained on the device and
# the host synchronises ONCE for the whole batch; steps behind a β <= tol are skipped on the device.
# Returns the number of steps done.  eigsolve's inner loop calls this instead of looping over expand!.
function expand_many!(iter::LanczosIterator{<:B200CSR}, state::LanczosFactorization, nsteps::Integer, tol::Real)
    iter.keepvecs || error("the fused Lanczos step keeps all Krylov vectors")
    V, r = state.V, state.r
    ctx, k = r.ctx, length(V)
    cols = Vector{Int32}(undef, k + nsteps + 1)
    for i in 1:k
        cols[i] = V[i].handle
    end
    cols[k + 1] = r.handle
    αs, βs = Vector{Float64}(undef, nsteps), Vector{Float64}(undef, nsteps)
    done, rout = Ref{Cint}(0), Ref{Int32}(0)
    tag, η = _tag(iter.orth)
    st = ccall((:b2k_lanczos_expand_many, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int32}, Cint, Cint, Float64, Float64, Cint, Float64, Ptr{Float64}, Ptr{Float64},
                Ref{Cint}, Ref{Int32}),
               ctx.h, iter.operator.h, cols, k, nsteps, normres(state), Float64(tol), tag, η, αs, βs, done, rout)
    d = Int(done[])
    if d > 0          # commit the completed steps BEFORE throwing (include/b200krylov.h, HANDLES)
        if cols[k + 1] == r.handle
            push!(V, r)                          # the residual's storage became the basis vector (lanczos.jl:257)
        else
            disown!(r)                           # the library released (and may have reused) that column
            push!(V, adopt(ctx, cols[k + 1]))
        end
        for i in 2:d
            push!(V, adopt(ctx, cols[k + i]))
        end
        state.r = adopt(ctx, rout[])
        append!(state.αs, αs[1:d]); append!(state.βs, βs[1:d])
        state.k += d
    end
    check(ctx.h, st)
    return d
end

# linsolve(::CG) — src/linsolve/cg.jl:62-101: one iteration = one call, p <- r + β p; q = A p (shifted);
# <p,q> in the SpMV epilogue; x += α p; r -= α q; ||r||² in the same sweep.  Returns (<p,q>, ||r||).
function cg_step!(A::B200CSR, x::B200Vec, r::B200Vec, p::B200Vec, q::B200Vec, α₀::Real, α₁::Real, β::Real, ρ::Real)
    pq, nr = Ref{Float64}(0), Ref{Float64}(0)
    check(x.ctx.h, ccall((:b2k_cg_step, lib), Cint,
                         (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32, Int32, Float64, Float64, Float64, Float64, Ref{Float64}, Ref{Float64}),
                         x.ctx.h, A.h, x.handle, r.handle, p.handle, q.handle, Float64(α₀), Float64(α₁), Float64(β), Float64(ρ), pq, nr))
    return pq[], nr[]
end
# linsolve(::BiCGStab) — src/linsolve/bicgstab.jl:95-150 in two calls (the half-step exit of :117-131 sits between):
#   half: p <- r + β(p − ω v) [first = true: p = r]; v = A p; σ = <r̃, v>; s = r − (ρ/σ) v; returns (σ, ||s||)
#   full: t = A s; ω = <t,s>/<t,t>; x += α p + ω s; r = s − ω t; returns (ω, ||r||, <r̃, r>)
function bicgstab_half!(A::B200CSR, r::B200Vec, rs::B200Vec, p::B200Vec, v::B200Vec, s::B200Vec,
                        α₀::Real, α₁::Real, β::Real, ω::Real, ρ::Real, first::Bool)
    σ, ns = Ref{Float64}(0), Ref{Float64}(0)
    check(r.ctx.h, ccall((:b2k_bicgstab_half, lib), Cint,
                         (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32, Int32, Int32, Float64, Float64, Float64, Float64, Float64, Cint,
                          Ref{Float64}, Ref{Float64}),
                         r.ctx.h, A.h, rs.handle, r.handle, p.handle, v.handle, s.handle, Float64(α₀), Float64(α₁), Float64(β),
                         Float64(ω), Float64(ρ), first ? 1 : 0, σ, ns))
    return σ[], ns[]
end
function bicgstab_full!(A::B200CSR, x::B200Vec, r::B200Vec, rs::B200Vec, p::B200Vec, s::B200Vec, t::B200Vec,
                        α₀::Real, α₁::Real, α::Real)
    ω, nr, ρ = Ref{Float64}(0), Ref{Float64}(0), Ref{Float64}(0)
    check(x.ctx.h, ccall((:b2k_bicgstab_full, lib), Cint,
                         (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32, Int32, Int32, Int32, Float64, Float64, Float64,
                          Ref{Float64}, Ref{Float64}, Ref{Float64}),
                         x.ctx.h, A.h, x.handle, r.handle, rs.handle, p.handle, s.handle, t.handle, Float64(α₀), Float64(α₁),
                         Float64(α), ω, nr, ρ))
    return ω[], nr[], ρ[]
end
# The same two loops with their iterations chained on the device (one host synchronisation per call): the scalar
# recurrences and the convergence tests of cg.jl:68 / bicgstab.jl:118,152 run in the kernels that produce the norms.
# cg_chain! returns (<p,q> per iteration, ||r|| per iteration); the iteration that met ||r|| < tol is the last.
function cg_chain!(A::B200CSR, x::B200Vec, r::B200Vec, p::B200Vec, q::B200Vec, α₀::Real, α₁::Real, β::Real, ρ::Real,
                   tol::Real, nsteps::Integer)
    pq, nr, done = zeros(Float64, nsteps), zeros(Float64, nsteps), Ref{Int32}(0)
    check(x.ctx.h, ccall((:b2k_cg_chain, lib), Cint,
                         (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32, Int32, Float64, Float64, Float64, Float64, Float64, Int32,
                          Ptr{Float64}, Ptr{Float64}, Ref{Int32}),
                         x.ctx.h, A.h, x.handle, r.handle, p.handle, q.handle, Float64(α₀), Float64(α₁), Float64(β), Float64(ρ),
                         Float64(tol), Int32(nsteps), pq, nr, done))
    return pq[1:done[]], nr[1:done[]]
end
# bicgstab_chain! returns an 8 × done matrix, one column per completed iteration:
# (ρ, σ, α, ||s||, ω, ||r||, next ρ, stop code); stop code 1: ||s|| < tol (the full step has not run), 2: ||r|| < tol.
function bicgstab_chain!(A::B200CSR, x::B200Vec, r::B200Vec, rs::B200Vec, p::B200Vec, v::B200Vec, s::B200Vec, t::B200Vec,
                         α₀::Real, α₁::Real, ρ::Real, ρold::Real, α::Real, ω::Real, tol::Real, nsteps::Integer)
    rec, done = zeros(Float64, 8, nsteps), Ref{Int32}(0)
    check(x.ctx.h, ccall((:b2k_bicgstab_chain, lib), Cint,
                         (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Int32, Int32, Int32, Int32, Int32, Float64, Float64, Float64,
                          Float64, Float64, Float64, Float64, Int32, Ptr{Float64}, Ref{Int32}),
                         x.ctx.h, A.h, x.handle, r.handle, rs.handle, p.handle, v.handle, s.handle, t.handle, Float64(α₀),
                         Float64(α₁), Float64(ρ), Float64(ρold), Float64(α), Float64(ω), Float64(tol), Int32(nsteps), rec, done))
    return rec[:, 1:done[]]
end
# KrylovKit.linsolve(A::B200CSR, b, x₀, alg::CG / BiCGStab, a₀, a₁) are the reference drivers (cg.jl, bicgstab.jl)
# with their loop bodies replaced by the calls above — krylovkit.jl_b200/linsolve.py::_cg/_bicgstab is that code,
# statement for statement, and is what the test-suite runs.

end # module
