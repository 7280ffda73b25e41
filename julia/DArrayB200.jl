# DArrayB200.jl -- reference-side binding for libdab200.so  (UNVERIFIED: there is no Julia in the build image; this file is the
# binding a DistributedArrays.jl maintainer would add, written against include/dab200.h; the executable stand-in used by the
# tests is the Python ctypes layer in distributedarrays.jl_b200/_lib.py, which binds the very same symbols).
#
# Idea: DistributedArrays.jl is generic in the chunk type `A` of `DArray{T,N,A}` (reference src/darray.jl:25).  `B200Array{T,N}`
# is a chunk type whose data lives in one GPU's HBM; it overloads exactly the Base generics the hot path calls on
# `localpart(d)`, so that the reference's own `map!` / broadcast / `mapreduce` / `mapreduce(...; dims)` code runs unchanged and
# lands in the CUDA kernels:
#
#   reference call site                                   Base generic overloaded here          C entry point
#   src/broadcast.jl:80  copyto!(localpart(dest), lbc)    Base.copyto!(::B200Array, ::Broadcasted)   dab_affine / dab_unary / dab_binary* / dab_broadcast_expr
#   src/broadcast.jl:96  copy(lbc)                        Base.copy(::Broadcasted{B200Style})        same + dab_alloc
#   src/mapreduce.jl:8   map!(f, localpart(dest), src)    Base.map!(f, ::B200Array, ::B200Array)     dab_affine / ...
#   src/mapreduce.jl:23,31 mapreduce(f, op, localpart)    Base.mapreduce / Base.reduce               dab_reduce_host
#   src/mapreduce.jl:64,77 mapreduce(...; dims)           Base.mapreducedim!                         dab_reducedim
#   src/mapreduce.jl:100-127 all/any/count/extrema        Base.all / any / count / extrema           dab_reduce_host
#   src/darray.jl:815    localpart(d)[idxs...]            Base.getindex(::B200Array, ranges...)      dab_copy_box
#   src/darray.jl:824,831 fill! / rand!                   Base.fill! / Random.rand!                  dab_fill / dab_rand_u01
#   src/mapreduce.jl:34  reduce(op, results)              (DArray method below)                      dab_mapreduce_all
#   src/linalg.jl:95-97,141 localpart(A)*xj, localpart(A)'*xj   Base.:*                                 dab_gemv
#   src/linalg.jl:1-17   transpose!(lp, rp)               LinearAlgebra.transpose! / adjoint!        dab_transpose_box
#   src/linalg.jl:1-17   adjoint!(lp, rp), complex T      LinearAlgebra.adjoint!                     dab_adjoint_box
#   src/sort.jl:8,22,61  sort(localpart(d)), sort!(lp)    Base.sort / Base.sort!                     dab_sort
#   src/sort.jl:8,22,61  sort(localpart(d); by = f)       sort_by (keys = f.(a) by broadcast)        dab_sort_by_key
#   (Base.sortperm: scalar getindex)  sortperm(localpart(d)), sortperm(d)   Base.sortperm (chunk and DVector methods)   dab_sort_pairs
#   (Base.sortperm: scalar getindex)  sortperm(A; dims)                    Base.sortperm(::DArray; dims), unverified   dab_sortperm_slices
#   src/mapreduce.jl:205 mapslices(f, localpart(y), dims) mapslices_sort / svdvals_batched       dab_sort_slices / dab_svdvals_batched
#   src/mapreduce.jl:315 _ppeval(f, localparts...; dim)   matmul_batched / eigvals_sym_batched  dab_matmul_batched / dab_eigvals_sym_batched
#                                                         ldiv_batched / det_batched            dab_ldiv_batched / dab_det_batched
#   (no reference method)  accumulate!(op, lp, lp; dims)   Base.accumulate! (cumsum! / cumprod!)   dab_scan
#   src/linalg.jl:95-97,141 localpart(A)*xj, SparseMatrixCSC chunks   Base.:* (SparseB200Chunk)   dab_spmv / dab_csc_to_csr
#   (Base._findmax: scalar getindex)  findmax(f, d) / findmin(f, d)   (DArray methods below)   dab_findminmax / dab_combine_findminmax
#   (Base getindex(A, I::AbstractArray): similar(d, axes(I)), src/darray.jl:238, scalar reads)  d[I::DArray{<:Integer}]
#                                                         Base.getindex(::DArray, ::DArray{<:Integer})   dab_index_gather
#   (Base getindex(A, I::AbstractArray{Bool}) / findall: scalar iteration)  d[m::DArray{Bool}], findall(m)
#                                                         Base.getindex(::DArray, ::DArray{Bool}), Base.findall   dab_compact_count / dab_compact
#   (Base.permutedims / permutedims!: scalar getindex)  permutedims(A, perm), permutedims!(dest, src, perm), unverified
#                                                         Base.permutedims / Base.permutedims!   dab_permute_box / dab_gather_box
module DArrayB200

using Distributed, DistributedArrays, LinearAlgebra
using LinearAlgebra: Adjoint, Transpose
import Base.Broadcast: Broadcasted, BroadcastStyle, AbstractArrayStyle

const libdab = get(ENV, "LIBDAB200", "libdab200.so")

# ---- status handling: mirror the reference's exception types -----------------------------------------------------------------
const DAB_OK = Int32(0)
function check(st::Int32, ctx::Ptr{Cvoid} = C_NULL)
    st == DAB_OK && return nothing
    msg = unsafe_string(ccall((:dab_last_error, libdab), Cstring, (Ptr{Cvoid},), ctx))
    st == 2 || st == 3 ? throw(ArgumentError(msg)) :
    st == 4 ? throw(DimensionMismatch(msg)) : throw(ErrorException("libdab200 [$st]: $msg"))
end

# ---- one context per worker process (one GPU per worker) ---------------------------------------------------------------------
const CTX = Ref{Ptr{Cvoid}}(C_NULL)
function ctx()
    if CTX[] == C_NULL
        ndev = Ref{Int32}(0)
        check(ccall((:dab_device_count, libdab), Int32, (Ref{Int32},), ndev))
        dev = Int32((myid() - 2 + ndev[]) % ndev[])           # worker pid 2 -> GPU 0, ...
        check(ccall((:dab_init, libdab), Int32, (Int32, Ref{Ptr{Cvoid}}), dev, CTX))
    end
    CTX[]
end

dab_dtype(::Type{Float32}) = Int32(0); dab_dtype(::Type{Float64}) = Int32(1)
dab_dtype(::Type{Int32}) = Int32(2);   dab_dtype(::Type{Int64}) = Int32(3); dab_dtype(::Type{Bool}) = Int32(4)
dab_dtype(::Type{ComplexF32}) = Int32(6); dab_dtype(::Type{ComplexF64}) = Int32(7)   # interleaved (re, im), Julia's own layout
dab_dtype(::Type{Float16}) = Int32(8)   # IEEE binary16

# ---- the chunk type ------------------------------------------------------------------------------------------------------------
mutable struct B200Array{T,N} <: AbstractArray{T,N}
    ptr::Ptr{Cvoid}
    dims::NTuple{N,Int}
    function B200Array{T,N}(::UndefInitializer, dims::NTuple{N,Int}) where {T,N}
        p = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:dab_alloc, libdab), Int32, (Ptr{Cvoid}, Csize_t, Ref{Ptr{Cvoid}}), ctx(), prod(dims) * sizeof(T), p), ctx())
        a = new{T,N}(p[], dims)
        finalizer(x -> ccall((:dab_free, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}), ctx(), x.ptr), a)   # cf. src/darray.jl:47-49
        a
    end
end
B200Array{T}(u::UndefInitializer, dims::Int...) where {T} = B200Array{T,length(dims)}(u, dims)
Base.size(a::B200Array) = a.dims
Base.similar(a::B200Array{T}, ::Type{S}, dims::Dims) where {T,S} = B200Array{S,length(dims)}(undef, dims)
Base.getindex(::B200Array, ::Int...) = error("scalar indexing of a B200Array is disabled (cf. DistributedArrays.allowscalar(false))")

# host <-> device  (distribute / Array(d): src/darray.jl:544-555, 574-582)
function B200Array(a::Array{T,N}) where {T,N}
    d = B200Array{T,N}(undef, size(a))
    check(ccall((:dab_h2d, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t), ctx(), d.ptr, a, sizeof(a)), ctx())
    check(ccall((:dab_sync, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx()); d
end
function Base.Array(d::B200Array{T,N}) where {T,N}
    a = Array{T,N}(undef, size(d))
    check(ccall((:dab_d2h, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t), ctx(), a, d.ptr, sizeof(a)), ctx())
    check(ccall((:dab_sync, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx()); a
end
Base.convert(::Type{B200Array{T,N}}, a::Array{T,N}) where {T,N} = B200Array(a)       # empty_localpart, src/darray.jl:62

function Base.fill!(a::B200Array{T}, x) where {T}                                       # src/darray.jl:822-827
    check(ccall((:dab_fill, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Ref{T}), ctx(), dab_dtype(T), a.ptr, length(a), T(x)), ctx()); a
end

# ---- elementwise: map! and in-place broadcast ------------------------------------------------------------------------------------
# A closure cannot cross the C ABI.  Known shapes are pattern-matched onto the hand-written kernels; any other Broadcasted tree is
# lowered to a C expression string and JIT-compiled by dab_broadcast_expr (NVRTC) -- `lower(bc)` below is the analogue of the
# Python tracer in distributedarrays.jl_b200/_broadcast.py.
struct Affine{T}; a::T; b::T; end                      # x -> a*x + b, two roundings (Julia never contracts to FMA)
(f::Affine)(x) = f.a * x + f.b

function Base.map!(f::Affine{T}, dest::B200Array{T}, src::B200Array{T}) where {T}       # src/mapreduce.jl:8
    length(dest) == length(src) || throw(DimensionMismatch("map!: lengths differ"))
    check(ccall((:dab_affine, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ref{T}, Ref{T}, Csize_t),
                ctx(), dab_dtype(T), dest.ptr, src.ptr, f.a, f.b, length(dest)), ctx()); dest
end

struct B200Style{N} <: AbstractArrayStyle{N} end
B200Style(::Val{N}) where {N} = B200Style{N}()
Base.Broadcast.BroadcastStyle(::Type{<:B200Array{T,N}}) where {T,N} = B200Style{N}()
Base.similar(bc::Broadcasted{B200Style{N}}, ::Type{T}) where {N,T} = B200Array{T,N}(undef, map(length, axes(bc)))

# y .= a .* x .+ b  ==  Broadcasted(+, (Broadcasted(*, (a, x)), b))                      # src/broadcast.jl:80
function Base.copyto!(dest::B200Array{T}, bc::Broadcasted{<:B200Style}) where {T}
    ab = match_affine(bc, T)
    if ab !== nothing
        a, x, b = ab
        return map!(Affine{T}(a, b), dest, x)
    end
    return broadcast_expr!(dest, bc)                    # general tree -> "jl_sub(a0, jl_mul(a1, jl_sin(a2)))" -> NVRTC
end
match_affine(bc, ::Type{T}) where {T} =
    (bc.f === (+) && length(bc.args) == 2 && bc.args[1] isa Broadcasted && bc.args[1].f === (*) &&
     bc.args[1].args[1] isa T && bc.args[1].args[2] isa B200Array{T} && bc.args[2] isa T) ?
        (bc.args[1].args[1], bc.args[1].args[2], bc.args[2]) : nothing
# General trees: walk the Broadcasted and emit the C expression dab_broadcast_expr compiles with NVRTC (the same lowering the
# Python tracer in distributedarrays.jl_b200/_broadcast.py performs; helper names are the jl_* functions of the JIT prelude).
const FN2 = Dict{Any,String}((+) => "jl_add", (-) => "jl_sub", (*) => "jl_mul", (/) => "jl_div", rem => "jl_rem", mod => "jl_mod",
                             div => "jl_idiv", max => "jl_max", min => "jl_min", (^) => "jl_pow", (<) => "jl_lt", (<=) => "jl_le",
                             (>) => "jl_gt", (>=) => "jl_ge", (==) => "jl_eq", (!=) => "jl_ne", (&) => "jl_and", (|) => "jl_or", xor => "jl_xor")
const FN1 = Dict{Any,String}((-) => "jl_neg", abs => "jl_abs", abs2 => "jl_abs2", sqrt => "jl_sqrt", inv => "jl_inv", floor => "jl_floor",
                             ceil => "jl_ceil", sign => "jl_sign", sin => "jl_sin", cos => "jl_cos", tan => "jl_tan", exp => "jl_exp",
                             log => "jl_log", tanh => "jl_tanh", isnan => "jl_isnan", identity => "")
ctype(::Type{Float32}) = "float"; ctype(::Type{Float64}) = "double"; ctype(::Type{Int32}) = "int"; ctype(::Type{Int64}) = "long long"; ctype(::Type{Bool}) = "bool"
ctype(::Type{Float16}) = "jl_f16"   # the NVRTC prelude's Float16 (widen to Float32, operate, round to Float16)
literal(x::Float32) = "__int_as_float((int)0x$(string(reinterpret(UInt32, x), base = 16)))"
literal(x::Float64) = "__longlong_as_double((long long)0x$(string(reinterpret(UInt64, x), base = 16))ULL)"
literal(x::Float16) = "jl_f16_bits((unsigned short)0x$(string(reinterpret(UInt16, x), base = 16)))"
literal(x::Integer) = "(($(ctype(typeof(x))))$(x))"
literal(x::Bool) = x ? "true" : "false"

# returns (expression string, element type); `args` collects the array / Ref-scalar leaves in order -> a0, a1, ...
function lower(bc::Broadcasted, args::Vector{Any})
    parts = [lower(a, args) for a in bc.args]
    Ts = map(last, parts)
    T = Base.promote_op(bc.f, Ts...)                                  # Julia's own result type: promotion stays exactly Julia's
    conv = [Ti === Tp ? s : "(($(ctype(Tp)))($s))" for ((s, Ti), Tp) in zip(parts, promote_types(bc.f, Ts, T))]
    name = length(conv) == 1 ? get(FN1, bc.f, nothing) : get(FN2, bc.f, nothing)
    name === nothing && error("DArrayB200: $(bc.f) is not served by the broadcast lowering (no host fallback)")
    (isempty(name) ? conv[1] : "$name($(join(conv, ", ")))", T)
end
lower(a::B200Array{T}, args) where {T} = (push!(args, a); ("a$(length(args) - 1)", T))
lower(x::Number, args) = (literal(x), typeof(x))
lower(r::Base.RefValue, args) = lower(r[], args)
# comparison / arithmetic operands are promoted to a common type first (Base.promote); bitwise and comparison results keep Bool
promote_types(f, Ts, T) = (f in (<, <=, >, >=, ==, !=)) ? fill(promote_type(Ts...), length(Ts)) : fill(T, length(Ts))

function broadcast_expr!(dest::B200Array{T,N}, bc::Broadcasted) where {T,N}
    args = Any[]
    expr, Tr = lower(bc, args)
    Tr === T || (expr = "(($(ctype(T)))($expr))")
    shape = Csize_t[size(dest)..., ones(Int, 4 - N)...]
    dense(sz) = Csize_t[cumprod([1; collect(sz)[1:end-1]])..., zeros(Int, 4 - length(sz))...]
    ostr = dense(size(dest)); ostr[N+1:end] .= 0
    strides = Csize_t[]
    for a in args                                                        # 0 = extruded dim (src/broadcast.jl:112-113)
        st = dense(size(a)); for d in 1:4; (d > ndims(a) || size(a, d) == 1) && (st[d] = 0); end; append!(strides, st)
    end
    check(ccall((:dab_broadcast_expr, libdab), Int32,
                (Ptr{Cvoid}, Cstring, Int32, Ptr{Cvoid}, Ptr{Csize_t}, Ptr{Csize_t}, Int32, Ptr{Int32}, Ptr{Ptr{Cvoid}}, Ptr{Csize_t}, Ptr{UInt64}),
                ctx(), expr, dab_dtype(T), dest.ptr, shape, ostr, length(args), Int32[dab_dtype(eltype(a)) for a in args],
                Ptr{Cvoid}[a.ptr for a in args], strides, zeros(UInt64, length(args))), ctx())
    dest
end

# ---- reductions --------------------------------------------------------------------------------------------------------------------
const OPS = Dict{Any,Int32}(Base.add_sum => 0, (+) => 0, Base.mul_prod => 1, (*) => 1, max => 2, min => 3)
const MAPS = Dict{Any,Int32}(identity => 0, abs => 1, abs2 => 2, (-) => 3)
result_type(::Type{T}, op, f = identity) where {T} = (T <: AbstractFloat || op >= 2) ? T : Int64          # add_sum / mul_prod widen Int32
# Complex{T}: sum / prod of z or -z are Complex{T}; abs / abs2 maps give T (the 16-byte slot holds re, im)
result_type(::Type{Complex{T}}, op, f = identity) where {T<:Union{Float32,Float64}} = (f === abs || f === abs2) ? T : Complex{T}

function Base.mapreduce(f, op, a::B200Array{T}; dims = :, init = nothing) where {T}         # src/mapreduce.jl:23,31,64
    haskey(OPS, op) && haskey(MAPS, f) || error("DArrayB200: mapreduce($f, $op) is not served by a kernel (no host fallback)")
    dims === Colon() || return mapreducedim(f, op, a, dims, init)
    out = zeros(UInt64, 2)
    check(ccall((:dab_reduce_host, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}),
                ctx(), dab_dtype(T), OPS[op], MAPS[f], C_NULL, a.ptr, length(a), out), ctx())
    reinterpret(result_type(T, OPS[op], f), out)[1]
end
Base.reduce(op, a::B200Array; kw...) = mapreduce(identity, op, a; kw...)

function mapreducedim(f, op, a::B200Array{T,N}, dims, init) where {T,N}
    region = Tuple(dims)
    all(d -> d >= 1, region) || throw(ArgumentError("region dimension(s) must be ≥ 1, got $dims"))
    rdims = ntuple(i -> i in region ? 1 : size(a, i), N)
    R = B200Array{result_type(T, OPS[op], f),N}(undef, rdims)   # complex T: SUM of z only (dab_reducedim refuses other ops / maps)
    init === nothing || fill!(R, init)
    # one (inner, reduce, outer) pass per maximal run of reduced dims; single leading / single trailing run shown
    k = findfirst(i -> !(i in region), 1:N)
    inner, red, outer = k === nothing ? (1, length(a), 1) :
                        (first(region) == 1 ? (1, prod(size(a)[1:k-1]), prod(size(a)[k:end])) :
                                              (prod(size(a)[1:first(region)-1]), prod(size(a)[collect(region)]), prod(size(a)[last(region)+1:end])))
    check(ccall((:dab_reducedim, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Int32),
                ctx(), dab_dtype(T), OPS[op], MAPS[f], a.ptr, inner, red, outer, R.ptr, init === nothing ? 0 : 1), ctx())
    R
end
Base.mapreducedim!(f, op, R::B200Array, A::B200Array) = (copyto!(R, mapreduce(f, op, A; dims = findall(size(R) .!= size(A)))); R)  # src/mapreduce.jl:77

# ---- scans: accumulate!(op, B, A; dims, init) on one chunk (base/accumulate.jl), ONE dab_scan launch ---------------------------------------------
# op in + * max min (add_sum / mul_prod reach here as + / * through cumsum! / cumprod!); eltype(B) must be the result type of dab_scan's table.
# init enters as the carry slab: inner*outer copies of init in the carrier type (dab_scan_carrier_dtype).  The cross-chunk carry of a DArray
# whose dims is split is the host runtime's job (distributedarrays.jl_b200/_scan.py); this method serves one chunk.
const SCAN_OPS = Dict{Any,Int32}(+ => 0, Base.add_sum => 0, * => 1, Base.mul_prod => 1, max => 2, min => 3)
carrier_type(code::Int32, ::Type{T}) where {T} = code == Int32(1) ? Float64 : code == Int32(3) ? Int64 : T
function Base.accumulate!(op, B::B200Array{R,N}, A::B200Array{T,N}; dims::Integer, init = nothing) where {R,T,N}
    haskey(SCAN_OPS, op) || error("DArrayB200: accumulate!($op) is not served by a kernel (no host fallback)")
    dims > 0 || throw(ArgumentError("dims must be a positive integer"))
    axes(B) == axes(A) || throw(DimensionMismatch("shape of B must match A"))
    dims > N && return copyto!(B, A)
    c = Ref{Int32}(0)
    check(ccall((:dab_scan_carrier_dtype, libdab), Int32, (Int32, Int32, Int32, Ref{Int32}), dab_dtype(T), SCAN_OPS[op], dab_dtype(R), c))
    inner, len, outer = prod(size(A)[1:dims-1]), size(A, dims), prod(size(A)[dims+1:end])
    carry = init === nothing ? nothing : fill!(B200Array{carrier_type(c[], T),1}(undef, (inner * outer,)), init)
    check(ccall((:dab_scan, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(T), SCAN_OPS[op], dab_dtype(R), A.ptr, inner, len, outer, carry === nothing ? C_NULL : carry.ptr, B.ptr), ctx())
    B
end

# ---- findmax / findmin (K20): ONE dab_findminmax launch per chunk; the chunk winners, made global through localindices, are folded by
# dab_combine_findminmax (any order: the winner is the largest order key, then the smallest global linear index).  The index is Julia's:
# an Int for a vector, a CartesianIndex otherwise.  Only DArrays of B200Array chunks with a served element type take these methods; every
# other DArray keeps Base's generic findmax.  f outside identity / abs / abs2 is mapped first (f.(d), the elementwise kernels), and the
# dims form is left to Base's generic findminmax! (the kernel-backed dims form is the host runtime's, distributedarrays.jl_b200/_findmax.py).
const FIND_MAPS = Dict{Any,Int32}(identity => 0, abs => 1, abs2 => 2)
const FindT = Union{Float32,Float64,Int32,Int64,Bool}
const FindDArray{T,N} = DArray{T,N,<:B200Array{T,N}}
function chunk_findminmax(a::B200Array{T}, which::Int32, f) where {T}
    slot = B200Array{UInt8,1}(undef, (16,))
    check(ccall((:dab_findminmax, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}),
                ctx(), dab_dtype(T), which, FIND_MAPS[f], C_NULL, a.ptr, length(a), slot.ptr), ctx())
    Array(slot)
end
function findminmax_darray(f, d::FindDArray{T,N}, which::Int32) where {T<:FindT,N}
    isempty(d) && throw(ArgumentError("reducing over an empty collection is not allowed"))
    recs = UInt8[]
    for (p, I) in zip(procs(d), d.indices)
        all(!isempty, I) || continue
        r = remotecall_fetch(() -> chunk_findminmax(localpart(d), which, f), p)
        li = reinterpret(Int64, r[9:16])[1]                                         # 0-based, chunk-local
        c = CartesianIndices(map(length, I))[li + 1]
        g = LinearIndices(size(d))[CartesianIndex(map((k, rng) -> first(rng) + k - 1, Tuple(c), I))]
        append!(recs, r[1:8], reinterpret(UInt8, [Int64(g)]))
    end
    out = zeros(UInt8, 16)
    check(ccall((:dab_combine_findminmax, libdab), Int32, (Int32, Int32, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}), dab_dtype(T), which, recs, length(recs) ÷ 16, out))
    v, g = reinterpret(T, out[1:sizeof(T)])[1], reinterpret(Int64, out[9:16])[1]
    v, N == 1 ? Int(g) : CartesianIndices(size(d))[g]
end
for (fn, which) in ((:findmax, Int32(0)), (:findmin, Int32(1)))
    @eval function Base.$fn(f, d::FindDArray{T}; dims = :) where {T<:FindT}
        dims isa Colon || return invoke(Base.$fn, Tuple{Any,AbstractArray}, f, d; dims = dims)
        haskey(FIND_MAPS, f) ? findminmax_darray(f, d, $which) : Base.$fn(identity, f.(d))
    end
    @eval Base.$fn(d::FindDArray{T}; dims = :) where {T<:FindT} = Base.$fn(identity, d; dims = dims)
end

# ---- SparseMatrixCSC chunks (UNVERIFIED, like the rest of this file): distribute(S) with a sparse S uploads each localpart as three device
# arrays; Julia's 1-based colptr / rowval become 0-based on upload.  localpart(A)*xj and localpart(A)'*xj (src/linalg.jl:95-97, 141) are
# SparseArrays' loops, i.e. dab_spmv on the row-major copy (built once by dab_csc_to_csr) or on the CSC arrays themselves.
using SparseArrays: SparseMatrixCSC, getcolptr, rowvals, nonzeros
mutable struct SparseB200Chunk{T} <: AbstractMatrix{T}
    m::Int; n::Int; nnz::Int
    colptr::B200Array{Int64,1}; rowval::B200Array{Int32,1}; nzval::B200Array{T,1}
    csr::Union{Nothing,Tuple{B200Array{Int64,1},B200Array{Int32,1},B200Array{T,1}}}
end
Base.size(a::SparseB200Chunk) = (a.m, a.n)
SparseArrays.nnz(a::SparseB200Chunk) = a.nnz
function SparseB200Chunk(S::SparseMatrixCSC{T}) where {T<:Union{Float32,Float64,Int32,Int64}}
    size(S, 1) <= typemax(Int32) || throw(ArgumentError("sparse chunks of more than 2^31-1 rows are not served"))
    SparseB200Chunk{T}(size(S)..., nnz(S), B200Array(Int64.(getcolptr(S) .- 1)), B200Array(Int32.(rowvals(S) .- 1)), B200Array(copy(nonzeros(S))), nothing)
end
function row_major!(a::SparseB200Chunk{T}) where {T}
    if a.csr === nothing
        rp, ci, v = B200Array{Int64,1}(undef, (a.m + 1,)), B200Array{Int32,1}(undef, (a.nnz,)), B200Array{T,1}(undef, (a.nnz,))
        check(ccall((:dab_csc_to_csr, libdab), Int32, (Ptr{Cvoid}, Int32, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
                    Ptr{Cvoid}, Ptr{Cvoid}), ctx(), dab_dtype(T), a.m, a.n, a.nnz, a.colptr.ptr, a.rowval.ptr, a.nzval.ptr, rp.ptr, ci.ptr, v.ptr), ctx())
        a.csr = (rp, ci, v)
    end
    a.csr
end
function spmv!(r::B200Array{T,1}, nrows, nnz, ptr, idx, val, x::B200Array{T,1}) where {T}
    check(ccall((:dab_spmv, libdab), Int32, (Ptr{Cvoid}, Int32, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(T), nrows, nnz, ptr.ptr, idx.ptr, val.ptr, x.ptr, r.ptr), ctx())
    r
end
function Base.:*(a::SparseB200Chunk{T}, x::B200Array{T,1}) where {T}
    rp, ci, v = row_major!(a)
    spmv!(B200Array{T,1}(undef, (a.m,)), a.m, a.nnz, rp, ci, v, x)
end
Base.:*(a::Union{Adjoint{T,<:SparseB200Chunk{T}},Transpose{T,<:SparseB200Chunk{T}}}, x::B200Array{T,1}) where {T<:Real} =
    (p = parent(a); spmv!(B200Array{T,1}(undef, (p.n,)), p.n, p.nnz, p.colptr, p.rowval, p.nzval, x))

# ---- the combine seam: sum(d::DArray{T,N,<:B200Array}) in ONE call per worker ----------------------------------------------------------
# replaces  results = asyncmap(procs(d)) do p; remotecall_fetch(...) end;  reduce(op, results)   (src/mapreduce.jl:29-35):
# every worker launches the fused kernel (chunk reduce + peer-memory all-gather + ordered fold); the caller fetches one scalar.
function Base._mapreduce(f, op, ::IndexCartesian, d::DArray{T,N,<:B200Array}) where {T,N}
    haskey(OPS, op) && haskey(MAPS, f) || error("DArrayB200: mapreduce($f, $op) is not served by a kernel")
    results = asyncmap(procs(d)) do p
        remotecall_fetch(p) do
            a = localpart(d); out = zeros(UInt64, 2)
            check(ccall((:dab_mapreduce_all, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}),
                        ctx(), dab_dtype(T), OPS[op], MAPS[f], C_NULL, a.ptr, length(a), out), ctx())
            reinterpret(result_type(T, OPS[op], f), out)[1]
        end
    end
    first(results)        # every worker already holds the left-folded result
end

# communicator / mailbox bring-up: rank 0 creates the NCCL id, the ids and IPC handles travel over Distributed (control plane only)
function init_comm(pids = workers())
    id = remotecall_fetch(pids[1]) do
        buf = zeros(UInt8, 128); check(ccall((:dab_comm_unique_id, libdab), Int32, (Ptr{UInt8},), buf)); buf
    end
    @sync for (r, p) in enumerate(pids)
        @async remotecall_wait(p) do
            check(ccall((:dab_comm_init_rank, libdab), Int32, (Ptr{Cvoid}, Ptr{UInt8}, Int32, Int32), ctx(), id, r - 1, length(pids)), ctx())
        end
    end
    handles = [remotecall_fetch(p) do
                   h = zeros(UInt8, 64); check(ccall((:dab_mailbox_create, libdab), Int32, (Ptr{Cvoid}, Ptr{UInt8}), ctx(), h), ctx()); h
               end for p in pids]
    allh = reduce(vcat, handles)
    @sync for (r, p) in enumerate(pids)
        @async remotecall_wait(p) do
            check(ccall((:dab_mailbox_attach, libdab), Int32, (Ptr{Cvoid}, Ptr{UInt8}, Int32, Int32), ctx(), allh, r - 1, length(pids)), ctx())
        end
    end
end

# ---- Level-2 and sort on the chunk type (widening rows): the generic code of src/linalg.jl and src/sort.jl then runs unchanged ------
# localpart(A)*xj  /  localpart(A)'*xj  inside mul!(y::DVector, A::DMatrix, x, α, β)  (src/linalg.jl:95-97, 141)
function gemv(trans::Bool, A::B200Array{T,2}, x::B200Array{T,1}) where {T}
    m, n = size(A)
    r = B200Array{T,1}(undef, (trans ? n : m,))
    check(ccall((:dab_gemv, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(T), trans ? 1 : 0, A.ptr, m, n, x.ptr, r.ptr), ctx())
    r
end
Base.:*(A::B200Array{T,2}, x::B200Array{T,1}) where {T} = gemv(false, A, x)
Base.:*(A::Adjoint{T,<:B200Array{T,2}}, x::B200Array{T,1}) where {T<:Real} = gemv(true, parent(A), x)
Base.:*(A::Transpose{T,<:B200Array{T,2}}, x::B200Array{T,1}) where {T} = gemv(true, parent(A), x)

# transpose!(lp, rp) / adjoint!(lp, rp) of copy(::Transpose{T,<:DArray{T,2}})  (src/linalg.jl:1-17), real T
function LinearAlgebra.transpose!(dst::B200Array{T,2}, src::B200Array{T,2}) where {T}
    rows, cols = size(src)
    check(ccall((:dab_transpose_box, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t),
                ctx(), sizeof(T), dst.ptr, cols, src.ptr, rows, rows, cols), ctx())
    dst
end
LinearAlgebra.adjoint!(dst::B200Array{T,2}, src::B200Array{T,2}) where {T<:Real} = transpose!(dst, src)
# adjoint!(lp, rp) of copy(::Adjoint{<:Complex,<:DArray})  (src/linalg.jl:1-17): transpose and conjugate in one pass
function LinearAlgebra.adjoint!(dst::B200Array{T,2}, src::B200Array{T,2}) where {T<:Union{ComplexF32,ComplexF64}}
    rows, cols = size(src)
    check(ccall((:dab_adjoint_box, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t),
                ctx(), dab_dtype(T), dst.ptr, cols, src.ptr, rows, rows, cols), ctx())
    dst
end

# sort(localpart(d)) / sort!(lp_sorting)  (src/sort.jl:8, 22, 61); keys only, isless order
function Base.sort!(a::B200Array{T,1}; kw...) where {T}
    tmp = B200Array{T,1}(undef, size(a))
    check(ccall((:dab_sort, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t),
                ctx(), dab_dtype(T), a.ptr, a.ptr, tmp.ptr, length(a)), ctx())
    a
end
function sort_keys(a::B200Array{T,1}) where {T}
    out = B200Array{T,1}(undef, size(a)); tmp = B200Array{T,1}(undef, size(a))
    check(ccall((:dab_sort, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t),
                ctx(), dab_dtype(T), a.ptr, out.ptr, tmp.ptr, length(a)), ctx())
    out
end

# sort(localpart(d); by = f) / sort!(lp_sorting; by = f)  (src/sort.jl:8, 22, 61 with the :by keyword of :111): keys = f.(a) through
# the broadcast lowering (one fused kernel), then the values are ordered stably by the keys (packed key|position words sorted by K11).
function sort_by(a::B200Array{T,1}, keys::B200Array{K,1}) where {T,K}
    n = length(a); need = Ref{Csize_t}(0)
    check(ccall((:dab_sort_by_key_scratch_bytes, libdab), Int32, (Int32, Csize_t, Ref{Csize_t}), dab_dtype(K), n, need), ctx())
    out = B200Array{T,1}(undef, size(a)); scratch = B200Array{UInt8,1}(undef, (Int(need[]),))
    check(ccall((:dab_sort_by_key, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t),
                ctx(), dab_dtype(K), keys.ptr, sizeof(T), a.ptr, out.ptr, scratch.ptr, need[], n), ctx())
    out
end
# keyword arguments do not take part in dispatch: ONE method serves both spellings
Base.sort(a::B200Array{T,1}; by = identity, kw...) where {T} = by === identity ? sort_keys(a) : sort_by(a, by.(a))

# K21: keys and Int64 values in the stable isless order of the keys (every NaN equal); vals === nothing means vals[i] = base + i.
# Returns (sorted keys, values).  keys and vals are not written.
function sort_pairs(keys::B200Array{K,1}, vals::Union{Nothing,B200Array{Int64,1}}, base::Int64) where {K}
    n = length(keys); need = Ref{Csize_t}(0)
    check(ccall((:dab_sort_pairs_scratch_bytes, libdab), Int32, (Int32, Csize_t, Ref{Csize_t}), dab_dtype(K), n, need), ctx())
    kout = B200Array{K,1}(undef, size(keys)); vout = B200Array{Int64,1}(undef, size(keys))
    scratch = B200Array{UInt8,1}(undef, (Int(need[]),))
    check(ccall((:dab_sort_pairs, libdab), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t),
                ctx(), dab_dtype(K), keys.ptr, kout.ptr, vals === nothing ? C_NULL : vals.ptr, base, vout.ptr, scratch.ptr, need[], n), ctx())
    kout, vout
end
# sortperm(localpart(d)): 1-based, stable; by = f orders by the keys f.(a) (one fused broadcast kernel)
Base.sortperm(a::B200Array{T,1}; by = identity, kw...) where {T} = sort_pairs(by === identity ? a : by.(a), nothing, Int64(1))[2]

# sortperm(d::DVector): K21 on every chunk with base = the chunk's first global index, then the sorted runs are merged on the caller
# in worker order (a stable merge: equal keys keep ascending global index) and the permutation is distributed over procs(d).  The
# Python runtime instead runs sort's samplesort with the index plane (the layout of sort(d)); this method keeps the binding small.
function Base.sortperm(d::DArray{T,1,B200Array{T,1}}; by = identity, kw...) where {T}
    runs = [remotecall_fetch(p) do
                a = localpart(d)
                k, v = sort_pairs(by === identity ? a : by.(a), nothing, Int64(first(localindices(d)[1])))
                Array(k), Array(v)
            end for p in procs(d)]
    keys = reduce(vcat, first.(runs)); idx = reduce(vcat, last.(runs))
    distribute(idx[sortperm(keys; alg = Base.Sort.DEFAULT_STABLE)]; procs = procs(d))
end

# sortperm(localpart(A); dims) with global indices (K26, unverified: no Julia run on a GPU yet): every fibre along `dims` of the chunk at
# 0-based offset `lo` in an array of size `gdims` gets the 1-based global LinearIndices of its elements in the stable isless order of
# `keys`; with `vals` the values are moved to the same places.  `dims` must be whole in the chunk.
function sortperm_slices(keys::B200Array{K,N}, dims::Integer, lo::NTuple{N,Int}, gdims::NTuple{N,Int};
                         vals::Union{Nothing,B200Array} = nothing) where {K,N}
    perm = B200Array{Int64,N}(undef, size(keys))
    vout = vals === nothing ? nothing : similar(vals)
    check(ccall((:dab_sortperm_slices, libdab), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int32, Ptr{Csize_t}, Ptr{Csize_t}, Ptr{Csize_t}, Int32, Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(K), keys.ptr, N, Csize_t[size(keys)...], Csize_t[lo...], Csize_t[gdims...], dims, perm.ptr,
                vals === nothing ? 0 : sizeof(eltype(vals)), vals === nothing ? C_NULL : vals.ptr, vout === nothing ? C_NULL : vout.ptr), ctx())
    perm, vout
end
# sortperm(A::DArray; dims): each worker runs K26 on its localpart when `dims` is whole there (the Python runtime also redistributes as
# mapslices does when it is split); the result has A's layout.
function Base.sortperm(A::DArray{T,N,B200Array{T,N}}; dims::Integer, by = identity, kw...) where {T,N}
    size(A.indices, dims) == 1 || throw(ArgumentError("sortperm(A; dims): dimension dims is split over workers; redistribute first"))
    DArray(size(A), procs(A), size(A.indices)) do I
        a = localpart(A)
        sortperm_slices(by === identity ? a : by.(a), dims, Tuple(first(r) - 1 for r in I), size(A))[1]
    end
end

# mapslices(f, localpart(y), dims=z)  (src/mapreduce.jl:205) for f = sort (one dim) and f = svdvals (two dims, slices already packed as
# `batch` column-major m x n matrices: the Python runtime packs them with dab_gather_box).  Julia's LAPACK wrapper rejects non-finite
# input (chkfinite); so does this one, once the status word has been read back.
function mapslices_sort(a::B200Array{T,N}, d::Int) where {T,N}
    out = B200Array{T,N}(undef, size(a))
    inner, len, outer = prod(size(a)[1:d-1]; init = 1), size(a, d), prod(size(a)[d+1:N]; init = 1)
    check(ccall((:dab_sort_slices, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t),
                ctx(), dab_dtype(T), a.ptr, out.ptr, inner, len, outer), ctx())
    out
end
function svdvals_batched(a::B200Array{T,3}) where {T<:Union{Float32,Float64}}
    m, n, batch = size(a)
    S = B200Array{T,2}(undef, (min(m, n), batch)); st = B200Array{Int32,1}(undef, (1,))
    check(ccall((:dab_svdvals_batched, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(T), a.ptr, m, n, batch, S.ptr, st.ptr), ctx())
    Array(st)[1] == 0 || throw(ArgumentError("matrix contains Infs or NaNs"))
    S
end

# _ppeval(f, localparts...; dim)  (src/mapreduce.jl:210-255) for f = * (slices already packed one after the other; a broadcast operand is
# passed with stride 0) and f = eigvals of real symmetric slices (packed as `batch` column-major n x n matrices).  A slice that is not
# exactly symmetric has complex eigenvalues in general: not served.
function matmul_batched(A::B200Array{T}, sa::Int, B::B200Array{T}, sb::Int, m::Int, n::Int, k::Int, batch::Int) where {T}
    C = B200Array{T,3}(undef, (m, n, batch))
    check(ccall((:dab_matmul_batched, libdab), Int32,
                (Ptr{Cvoid}, Int32, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t),
                ctx(), dab_dtype(T), m, n, k, A.ptr, sa, B.ptr, sb, C.ptr, batch), ctx())
    C
end
function eigvals_sym_batched(a::B200Array{T,3}) where {T<:Union{Float32,Float64}}
    n, n2, batch = size(a)
    n == n2 || throw(DimensionMismatch("matrix is not square: dimensions are ($n, $n2)"))
    W = B200Array{T,2}(undef, (n, batch)); st = B200Array{Int32,1}(undef, (1,))
    check(ccall((:dab_eigvals_sym_batched, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}),
                ctx(), dab_dtype(T), a.ptr, n, batch, W.ptr, st.ptr), ctx())
    flags = Array(st)[1]
    flags & 1 == 0 || throw(ArgumentError("matrix contains Infs or NaNs"))
    flags & 2 == 0 || error("eigvals: a slice is not symmetric; complex eigenvalues are not served")
    W
end

# _ppeval(f, localparts...; dim) for f = \ and f = det (K27): `batch` packed column-major n x n slices, n <= 64, stride 0 broadcasts.
# The status word names the lowest failing slice: (b << 8) | info, or | 0x80 for a NaN / Inf on the LU path.
function ldiv_batched(A::B200Array{T}, sa::Int, B::B200Array{T}, sb::Int, n::Int, nrhs::Int, batch::Int) where {T<:Union{Float32,Float64}}
    X = B200Array{T,3}(undef, (n, nrhs, batch)); st = B200Array{UInt64,1}(undef, (1,))
    check(ccall((:dab_ldiv_batched, libdab), Int32,
                (Ptr{Cvoid}, Int32, Csize_t, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}),
                ctx(), dab_dtype(T), n, nrhs, A.ptr, sa, B.ptr, sb, X.ptr, batch, st.ptr), ctx())
    w = Array(st)[1]
    w == typemax(UInt64) || (w & 0xff == 0x80 ? throw(ArgumentError("matrix contains Infs or NaNs")) : throw(SingularException(Int(w & 0xff))))
    X
end
function det_batched(a::B200Array{T,3}) where {T<:Union{Float32,Float64}}
    n, n2, batch = size(a)
    n == n2 || throw(DimensionMismatch("matrix is not square: dimensions are ($n, $n2)"))
    D = B200Array{T,1}(undef, (batch,))
    check(ccall((:dab_det_batched, libdab), Int32, (Ptr{Cvoid}, Int32, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t),
                ctx(), dab_dtype(T), n, a.ptr, n * n, D.ptr, batch), ctx())
    D
end

# localpart(A) * Bjk, transpose(localpart(A)) * Bjk inside _matmatmul!  (src/linalg.jl:218-226): K12, wgmma 3xTF32 for Float32
function gemm(transA::Bool, A::B200Array{T,2}, B::B200Array{T,2}) where {T}
    m, k = transA ? reverse(size(A)) : size(A)
    size(B, 1) == k || throw(DimensionMismatch("matrix A has dimensions ($m, $k), matrix B has dimensions $(size(B))"))
    R = B200Array{T,2}(undef, (m, size(B, 2)))
    check(ccall((:dab_gemm, libdab), Int32,
                (Ptr{Cvoid}, Int32, Int32, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}, Csize_t),
                ctx(), dab_dtype(T), transA, m, size(B, 2), k, A.ptr, size(A, 1), B.ptr, size(B, 1), R.ptr, m), ctx())
    R
end
Base.:*(A::B200Array{T,2}, B::B200Array{T,2}) where {T} = gemm(false, A, B)
Base.:*(A::Adjoint{T,<:B200Array{T,2}}, B::B200Array{T,2}) where {T<:Real} = gemm(true, parent(A), B)
Base.:*(A::Transpose{T,<:B200Array{T,2}}, B::B200Array{T,2}) where {T} = gemm(true, parent(A), B)

# add!(localpart(y), R[i,j], alpha) for all j after the beta scaling (src/linalg.jl:62-76, 101-117, 232-252): one fused launch over the
# stack of tile results that the producers PUT into this worker's exchange arena; dab_peer_barrier orders the puts (device side)
function accumulate_stack!(y::B200Array{T}, beta, alpha, stack::Ptr{Cvoid}, count::Integer) where {T}
    check(ccall((:dab_accumulate_stack, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Csize_t, Ref{T}, Ref{T}, Ptr{Cvoid}, Csize_t, Int32),
                ctx(), dab_dtype(T), y.ptr, length(y), T(beta), T(alpha), stack, length(y), count), ctx())
    y
end
peer_barrier() = check(ccall((:dab_peer_barrier, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx())

# localpart(d)[idxs...] with StepRange / Vector{Int} indices (src/darray.jl:661, 798-820): strided / table-driven gather
function Base.getindex(a::B200Array{T,N}, I::Vararg{Union{AbstractRange{Int},Vector{Int}},N}) where {T,N}
    out = B200Array{T,N}(undef, map(length, I))
    sstr = cumprod((1, size(a)[1:end-1]...)); dstr = cumprod((1, size(out)[1:end-1]...))
    tabs = [B200Array(Int64.((collect(I[k]) .- first(I[k])) .* sstr[k])) for k in 1:N]       # source offsets as tables (affine ones could pass strides)
    src = a.ptr + (sum((first(I[k]) - 1) * sstr[k] for k in 1:N)) * sizeof(T)
    check(ccall((:dab_gather_box, libdab), Int32,
                (Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Ptr{Clonglong}, Ptr{Ptr{Cvoid}}, Ptr{Cvoid}, Ptr{Clonglong}, Ptr{Ptr{Cvoid}}, Ptr{Csize_t}),
                ctx(), sizeof(T), N, out.ptr, Clonglong[dstr...], C_NULL, src, zeros(Clonglong, N), Ptr{Cvoid}[t.ptr for t in tabs],
                Csize_t[length.(I)...]), ctx())
    out
end

# d[I::DArray{<:Integer}] (Base's generic getindex: similar(d, axes(I)), src/darray.jl:238, filled by scalar reads): K22 on every
# localpart of R = similar(d, size(I)).  I[k] is a 1-based column-major linear index into d.  Every worker of R maps the other
# workers' localparts of d over CUDA IPC and reads its block of I with the reference's halo getindex (src/darray.jl:798-820), which
# brings the block through the host (the Python runtime copies it device to device); bad positions come back by remotecall_fetch.
# Peer mappings are cached per handle on each worker, as in the Python runtime, and released by ipc_close_all() (call it before
# the owners free their localparts, e.g. when the worker shuts down).
const IPC_MAPS = Dict{Vector{UInt8},Ptr{Cvoid}}()
function ipc_handle(a::B200Array)
    h = zeros(UInt8, 64)
    length(a) == 0 || check(ccall((:dab_ipc_get_handle, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{UInt8}), ctx(), a.ptr, h), ctx())
    h
end
ipc_open(h::Vector{UInt8}) = get!(IPC_MAPS, h) do
    p = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:dab_ipc_open, libdab), Int32, (Ptr{Cvoid}, Ptr{UInt8}, Ref{Ptr{Cvoid}}), ctx(), h, p), ctx())
    p[]
end
function ipc_close_all()
    for p in values(IPC_MAPS)
        check(ccall((:dab_ipc_close, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}), ctx(), p), ctx())
    end
    empty!(IPC_MAPS)
end
function Base.getindex(d::DArray{T,N,B200Array{T,N}}, I::DArray{<:Integer}) where {T,N}
    eltype(I) <: Union{Int32,Int64} || throw(ArgumentError("index element type $(eltype(I)) is not served (Int32, Int64)"))
    R = similar(d, size(I))
    owners = vec(d.pids)
    handles = Dict(p => remotecall_fetch(() -> ipc_handle(localpart(d)), p) for p in owners)
    # 0-based chunk starts from the chunk extents (an empty chunk repeats a cut), then size(d, k)
    cuts = reduce(vcat, [cumsum([0; [length(d.indices[ntuple(j -> j == k ? c : 1, N)...][k]) for c in 1:size(d.pids, k)]]) for k in 1:N])
    bad = asyncmap(procs(R)) do p
        remotecall_fetch(p) do
            J = localindices(R)
            ptrs = Ptr{Cvoid}[any(isempty, d.indices[c]) ? C_NULL : q == myid() ? localpart(d).ptr : ipc_open(handles[q])
                              for (c, q) in enumerate(owners)]
            blk = B200Array(Array(I[J...]))                                   # the halo read of I's block, uploaded
            pos = B200Array(fill(typemax(UInt64), 1))
            check(ccall((:dab_index_gather, libdab), Int32,
                        (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Csize_t, Int32, Ptr{Csize_t}, Ptr{Int32}, Ptr{Csize_t},
                         Ptr{Ptr{Cvoid}}, Ptr{Cvoid}),
                        ctx(), sizeof(T), localpart(R).ptr, blk.ptr, dab_dtype(eltype(I)), length(blk), N, Csize_t[size(d)...],
                        Int32[size(d.pids)...], Csize_t[cuts...], ptrs, pos.ptr), ctx())
            b = Array(pos)[1]
            b == typemax(UInt64) ? nothing : (LinearIndices(size(I))[CartesianIndex(Tuple(CartesianIndices(map(length, J))[b + 1]) .+ first.(J) .- 1)])
        end
    end
    found = filter(!isnothing, bad)
    isempty(found) || (close(R); throw(BoundsError(d, I[minimum(found)])))
    R
end

# d[m::DArray{Bool}] and findall(m) (Base's generic methods iterate element by element): K23 on every localpart of d, DESIGN.md §3.10.
# A run of a chunk is contiguous in the global column-major order; with k the first split dimension, chunk c has runs of
# prod(size(d)[1:k-1]) * ext[k] elements, run ids b + grid[k] * o and first linear indices inner * (start_k + size(d, k) * o).  Phase
# 1 counts tiles and scans them on each owner (the tables wait in COMPACT_PLANS), the host lays out the run offsets, phase 2 writes
# the selected elements into R's localparts through peer mappings.
const COMPACT_PLANS = Dict{Tuple{UInt,Int},Any}()
function compact_runs(d::DArray)
    dims, grid = size(d), size(d.pids)
    k = something(findfirst(>(1), grid), length(dims))
    inner, outer = prod(dims[1:k-1]), dims[k+1:end]
    runs = map(enumerate(d.indices)) do (c, I)
        ext = map(length, I)
        os = Int64[LinearIndices(outer)[CartesianIndex(Tuple(o) .+ first.(I[k+1:end]) .- 1)] - 1 for o in CartesianIndices(ext[k+1:end])]
        (inner * ext[k], ((c - 1) % grid[k]) .+ grid[k] .* os, inner .* (first(I[k]) - 1) .+ inner * dims[k] .* os)
    end
    runs, grid[k] * prod(outer)
end
function compact(d::DArray{T,N,B200Array{T,N}}, m::DArray{Bool,N}, index::Bool) where {T,N}
    size(m) == size(d) || throw(ArgumentError("logical indexing with a DArray{Bool} of other dims is not served"))
    runs, nruns = compact_runs(d)
    owners, key = vec(d.pids), objectid(d)
    tots = asyncmap(enumerate(owners)) do (c, p)
        remotecall_fetch(p) do
            run_len, ids, _ = runs[c]
            run_len * length(ids) == 0 && return zeros(Int64, length(ids))
            blk = B200Array(Array(m[d.indices[c]...]))                        # the halo read of the mask block, uploaded
            tiles = cld(run_len, 4096) * length(ids)
            counts, incl, tot = B200Array(zeros(Int32, tiles)), B200Array(zeros(Int64, tiles)), B200Array(zeros(Int64, length(ids)))
            check(ccall((:dab_compact_count, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t, Ptr{Cvoid}), ctx(), blk.ptr, run_len,
                        length(ids), counts.ptr), ctx())
            tpr, nr = tiles ÷ length(ids), length(ids)                         # Int32 SUM -> Int64 along each run of the tile table
            check(ccall((:dab_scan, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}),
                        ctx(), dab_dtype(Int32), Int32(0), dab_dtype(Int64), counts.ptr, 1, tpr, nr, C_NULL, incl.ptr), ctx())
            check(ccall((:dab_scan_totals, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Cvoid}, Csize_t, Csize_t, Csize_t, Ptr{Cvoid}),
                        ctx(), dab_dtype(Int32), Int32(0), dab_dtype(Int64), counts.ptr, 1, tpr, nr, tot.ptr), ctx())
            COMPACT_PLANS[(key, c)] = (blk, incl)
            Array(tot)
        end
    end
    totals = zeros(Int64, nruns)
    for (c, t) in enumerate(tots)
        totals[runs[c][2] .+ 1] .= t
    end
    offsets = [0; cumsum(totals)]
    R = similar(d, index ? Int64 : T, (offsets[end],))
    offsets[end] == 0 && return R
    handles = Dict(p => remotecall_fetch(() -> ipc_handle(localpart(R)), p) for p in procs(R))
    cuts = Csize_t[0; cumsum([length(I[1]) for I in vec(R.indices)])]
    asyncmap(enumerate(owners)) do (c, p)
        remotecall_fetch(p) do
            plan = pop!(COMPACT_PLANS, (key, c), nothing)
            plan === nothing && return nothing
            run_len, ids, lin = runs[c]
            info = B200Array(vec(permutedims([offsets[ids .+ 1] lin])))
            ptrs = Ptr{Cvoid}[isempty(R.indices[j][1]) ? C_NULL : q == myid() ? localpart(R).ptr : ipc_open(handles[q])
                              for (j, q) in enumerate(vec(R.pids))]
            check(ccall((:dab_compact, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid},
                        Int32, Ptr{Csize_t}, Ptr{Ptr{Cvoid}}), ctx(), index ? 0 : sizeof(T), plan[1].ptr, index ? C_NULL : localpart(d).ptr,
                        run_len, length(ids), plan[2].ptr, info.ptr, length(ptrs), cuts, ptrs), ctx())
            check(ccall((:dab_sync, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx())   # the peer stores have landed before R is read
            nothing
        end
    end
    R
end
Base.getindex(d::DArray{T,N,B200Array{T,N}}, m::DArray{Bool,N}) where {T,N} = compact(d, m, false)
Base.findall(m::DArray{Bool,N,B200Array{Bool,N}}) where {N} = compact(m, m, true)   # linear indices, on the devices (DESIGN.md §3.10)

# d[I::DArray{<:Integer}] = v (row f14; Base's setindex! writes one element per remote call): K24, DESIGN.md §3.11.  Unverified, as
# the K22 / K23 bindings.  Every owner of a chunk of I checks its block against per-chunk bitmaps of d (peer atomics), the host combines
# the flags (BoundsError before any store), duplicates take a winner table, then every owner stores its block through peer mappings.
function Base.setindex!(d::DArray{T,N,B200Array{T,N}}, v, I::DArray{<:Integer}) where {T,N}
    eltype(I) <: Union{Int32,Int64} || throw(ArgumentError("index element type $(eltype(I)) is not served (Int32, Int64)"))
    v isa Number || filter(!=(1), size(v)) == filter(!=(1), size(I)) || throw(DimensionMismatch("tried to assign $(size(v)) to $(size(I))"))
    isempty(I) && return d
    owners = vec(d.pids)
    lens = [prod(map(length, J)) for J in vec(d.indices)]
    cuts = reduce(vcat, [cumsum([0; [length(d.indices[ntuple(j -> j == k ? c : 1, N)...][k]) for c in 1:size(d.pids, k)]]) for k in 1:N])
    tab(n) = Dict(p => remotecall_fetch(() -> (t = B200Array(zeros(Int32, n(lens[c]))); (t, ipc_handle(t))), p) for (c, p) in enumerate(owners))
    ptrs(h, get) = Ptr{Cvoid}[lens[c] == 0 ? C_NULL : q == myid() ? get(q) : ipc_open(h[q][2]) for (c, q) in enumerate(owners)]
    dh = Dict(p => remotecall_fetch(() -> ipc_handle(localpart(d)), p) for p in owners)
    bits = tab(n -> cld(n, 32))
    vals = v isa Number ? nothing : reshape(collect(v), size(I))
    sig = (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Csize_t, Int32, Ptr{Csize_t}, Ptr{Int32}, Ptr{Csize_t}, Ptr{Ptr{Cvoid}}, Ptr{Cvoid})
    flags = asyncmap(procs(I)) do p
        remotecall_fetch(p) do
            J = localindices(I)
            any(isempty, J) && return (nothing, 0)
            st = B200Array(UInt64[typemax(UInt64), 0])
            check(ccall((:dab_scatter_check, libdab), Int32, sig, ctx(), localpart(I).ptr, dab_dtype(eltype(I)), length(localpart(I)), N,
                        Csize_t[size(d)...], Int32[size(d.pids)...], Csize_t[cuts...], ptrs(bits, q -> bits[q][1].ptr), st.ptr), ctx())
            b, dup = Array(st)
            (b == typemax(UInt64) ? nothing : LinearIndices(size(I))[CartesianIndex(Tuple(CartesianIndices(map(length, J))[b + 1]) .+ first.(J) .- 1)], dup)
        end
    end
    found = filter(!isnothing, first.(flags))
    isempty(found) || throw(BoundsError(d, I[minimum(found)]))
    dup = any(f -> f[2] != 0, flags)
    length(I) < 2^32 || !dup || throw(ArgumentError("8-byte winner tables are served by the Python host runtime only"))
    win = dup ? tab(identity) : nothing
    for phase in (dup ? (:winners, :store) : (:store,))
        asyncmap(procs(I)) do p
            remotecall_fetch(p) do
                J = localindices(I)
                any(isempty, J) && return nothing
                lin = B200Array([LinearIndices(size(I))[CartesianIndex(first(J[1]), Tuple(o)...)] - 1
                                 for o in CartesianIndices(map(length, J[2:end])) .+ CartesianIndex(first.(J[2:end]) .- 1)])
                wp = dup ? ptrs(win, q -> win[q][1].ptr) : Ptr{Cvoid}[]
                if phase === :winners
                    check(ccall((:dab_scatter_winners, libdab), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Csize_t, Csize_t, Ptr{Cvoid}, Int32, Int32,
                                Ptr{Csize_t}, Ptr{Int32}, Ptr{Csize_t}, Ptr{Ptr{Cvoid}}), ctx(), localpart(I).ptr, dab_dtype(eltype(I)),
                                length(localpart(I)), length(J[1]), lin.ptr, 4, N, Csize_t[size(d)...], Int32[size(d.pids)...], Csize_t[cuts...], wp), ctx())
                else
                    blk = vals === nothing ? nothing : B200Array(convert(Array{T}, vals[J...]))
                    x = Ref{T}(v isa Number ? convert(T, v) : zero(T))
                    check(ccall((:dab_scatter, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int32, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t,
                                Ptr{Cvoid}, Int32, Int32, Ptr{Csize_t}, Ptr{Int32}, Ptr{Csize_t}, Ptr{Ptr{Cvoid}}, Ptr{Ptr{Cvoid}}), ctx(), sizeof(T),
                                localpart(I).ptr, dab_dtype(eltype(I)), length(localpart(I)), blk === nothing ? C_NULL : blk.ptr, x, length(J[1]),
                                lin.ptr, dup ? 4 : 0, N, Csize_t[size(d)...], Int32[size(d.pids)...], Csize_t[cuts...],
                                ptrs(dh, q -> localpart(d).ptr), dup ? wp : C_NULL), ctx())
                end
                check(ccall((:dab_sync, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx())   # the peer atomics / stores have landed
                nothing
            end
        end
    end
    d
end

# d[m::DArray{Bool}] .= x (row f14): K25's scalar mode on every localpart of d, no plan.  Unverified.
function Base.setindex!(d::DArray{T,N,B200Array{T,N}}, x::Number, m::DArray{Bool,N}) where {T,N}
    size(m) == size(d) || throw(ArgumentError("logical indexing with a DArray{Bool} of other dims is not served"))
    asyncmap(vec(d.pids)) do p
        remotecall_fetch(p) do
            L = localpart(d)
            isempty(L) && return nothing
            blk = B200Array(Array(m[localindices(d)...]))                       # the halo read of the mask block, uploaded
            s = Ref{T}(convert(T, x))
            check(ccall((:dab_expand, libdab), Int32, (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Csize_t, Ptr{Cvoid}, Ptr{Cvoid}, Int32,
                        Ptr{Csize_t}, Ptr{Ptr{Cvoid}}, Ptr{Cvoid}), ctx(), sizeof(T), blk.ptr, L.ptr, length(L), 1, C_NULL, C_NULL, 0, C_NULL, C_NULL, s), ctx())
            nothing
        end
    end
    d
end

# permutedims(A, perm) / permutedims!(dest, src, perm) (row f18; Base's generic methods read a DArray with one scalar getindex per
# element): every worker of dest fills its localpart from the pieces of src its preimage box meets (local or CUDA-IPC peer loads), one
# launch per piece: dab_permute_box (K28), or dab_gather_box when dest's dim 1 is also contiguous in src (a batch of contiguous runs)
# or the plane of the two contiguous dims is below the measured size.
# Per piece the extent-1 dims are dropped and dest-adjacent dims contiguous on both sides merged, as permute_plan does in the Python
# runtime.  A matrix with perm (2, 1) is copy(transpose(A)).  Unverified: no Julia run on a GPU yet.
const PERMUTE_MIN_PLANE = Dict(1 => 1536, 2 => 512, 4 => 1024, 8 => 512, 16 => 512)   # below it a K28 tile is mostly idle (_permute.py)
function permute_collapse(ext, ds, ss)
    out = [[e, d, s] for (e, d, s) in zip(ext, ds, ss) if e != 1]
    isempty(out) && return ([1], [1], [1])
    merged = [out[1]]
    for (e, d, s) in out[2:end]
        pe, pd, ps = merged[end]
        d == pd * pe && s == ps * pe ? (merged[end][1] = pe * e) : push!(merged, [e, d, s])
    end
    (getindex.(merged, 1), getindex.(merged, 2), getindex.(merged, 3))
end
function Base.permutedims!(dest::DArray{T,N,B200Array{T,N}}, src::DArray{T,N,B200Array{T,N}}, perm) where {T,N}
    length(perm) == N || throw(ArgumentError("expected permutation of size $N, but length(perm)=$(length(perm))"))
    isperm(perm) || throw(ArgumentError("input is not a permutation"))
    all(size(dest, k) == size(src, perm[k]) for k in 1:N) || throw(DimensionMismatch("destination tensor of incorrect size"))
    dest === src && throw(ArgumentError("permutedims!: dest and src share storage (the result would be unspecified)"))
    owners = vec(src.pids)
    handles = Dict(p => remotecall_fetch(() -> ipc_handle(localpart(src)), p) for p in owners)
    asyncmap(procs(dest)) do p
        remotecall_fetch(p) do
            I = localindices(dest)
            any(isempty, I) && return nothing
            J = Vector{UnitRange{Int}}(undef, N)
            for k in 1:N
                J[perm[k]] = I[k]                                             # the preimage box in src
            end
            dstr = cumprod((1, map(length, I)[1:end-1]...))
            for (c, q) in enumerate(owners)
                K = src.indices[c]
                box = map(intersect, J, K)
                any(isempty, box) && continue
                sstr = cumprod((1, map(length, K)[1:end-1]...))
                sp = (q == myid() ? localpart(src).ptr : ipc_open(handles[q])) + sum((first(box[j]) - first(K[j])) * sstr[j] for j in 1:N) * sizeof(T)
                dp = localpart(dest).ptr + sum((first(box[perm[k]]) - first(J[perm[k]])) * dstr[k] for k in 1:N) * sizeof(T)
                e, ds, ss = permute_collapse([length(box[perm[k]]) for k in 1:N], collect(dstr), [sstr[perm[k]] for k in 1:N])
                n = length(e)
                q = n >= 2 && ds[1] == 1 && count(==(1), ss[2:end]) == 1 ? findlast(==(1), ss) : 0
                if q > 0 && e[1] * e[q] >= PERMUTE_MIN_PLANE[sizeof(T)] && min(e[1], e[q]) * sizeof(T) >= 16
                    check(ccall((:dab_permute_box, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Ptr{Clonglong}, Ptr{Cvoid}, Ptr{Clonglong},
                                Ptr{Csize_t}), ctx(), sizeof(T), n, dp, Clonglong[ds...], sp, Clonglong[ss...], Csize_t[e...]), ctx())
                else
                    check(ccall((:dab_gather_box, libdab), Int32, (Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Ptr{Clonglong}, Ptr{Ptr{Cvoid}}, Ptr{Cvoid},
                                Ptr{Clonglong}, Ptr{Ptr{Cvoid}}, Ptr{Csize_t}), ctx(), sizeof(T), n, dp, Clonglong[ds...], C_NULL, sp,
                                Clonglong[ss...], C_NULL, Csize_t[e...]), ctx())
                end
            end
            check(ccall((:dab_sync, libdab), Int32, (Ptr{Cvoid},), ctx()), ctx())       # the peer reads end before the owners move on
            nothing
        end
    end
    dest
end
Base.permutedims(A::DArray{T,N,B200Array{T,N}}, perm) where {T,N} =
    N == 2 && Tuple(perm) == (2, 1) ? copy(transpose(A)) :
    permutedims!(DArray(I -> B200Array{T,N}(undef, map(length, I)), ntuple(k -> size(A, perm[k]), N), procs(A)), A, perm)

# user code is then unchanged:
#   d = DArray(I -> B200Array(rand(Float32, map(length, I))), (8 * 2^30,))
#   d .= 1.5f0 .* d .+ 0.25f0 ;  map!(Affine(2f0, 1f0), d, d) ;  sum(d) ;  maximum(d) ;  sum(d2, dims = 1) ;  A * B ;  A' * x ;  sort(v)
end # module
