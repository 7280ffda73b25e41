/*
 * dab200.h -- C ABI of libdab200.so: the H100 (sm_90a) backend for the DArray
 *             map!/broadcast + mapreduce hot path of DistributedArrays.jl.
 *
 * The reference (DistributedArrays.jl v0.6.9) is pure Julia and has NO FFI / plugin
 * interface; this boundary is created at the two seams the reference already has
 * (SURVEY.md section 8b):
 *   1. the chunk-type seam  DArray{T,N,A}  (src/darray.jl:25)  -- a Julia chunk type
 *      B200Array{T,N} overloads the Base generics the hot path calls on localpart(d)
 *      and forwards them with ccall to the entry points below;
 *   2. the combine seam     reduce(op, results) (src/mapreduce.jl:34),
 *      mapreducedim_between! (src/mapreduce.jl:71-81), chunk()/setindex! slab fetch
 *      (src/darray.jl:458,798-820) -- replaced by the comm / peer entry points.
 * Every entry point cites the reference call site(s) it replaces.  Citations are relative
 * to the reference tree.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes.  Device pointers are raw CUDA device addresses
 *     (what a Julia B200Array would hold in a Ptr{Cvoid} field); host pointers are ordinary.
 *   - every function returns an int32_t status (DAB_OK == 0).  No C++ exception or sticky
 *     CUDA error crosses the ABI; dab_last_error(ctx) gives the text.
 *   - a dab_ctx is bound to ONE device and owns ONE stream.  The reference runs one
 *     single-threaded Julia process per worker (src/mapreduce.jl:6-10): one ctx per
 *     worker process.  All compute entry points are ASYNCHRONOUS on the ctx stream
 *     (== remotecall); dab_sync, events and the *_host variants are the sync points
 *     (== remotecall_wait / remotecall_fetch).  A ctx must not be used from two threads
 *     at once; different ctxs are independent.
 *   - a compute call is queued on the ctx stream no later than the next call on that ctx.
 *     dab_affine may be held back until then, so that a following dab_reduce /
 *     dab_reduce_host / dab_mapreduce_all of its output (same pointer, n and dtype, MAP_ID,
 *     SUM/PROD/MAX/MIN) runs as ONE kernel that stores y and reduces it; results are
 *     bit-identical either way.  dab_launch_count counts the held-back call as launched.
 *     dab_stream turns this off for the rest of the ctx's life (work queued directly on
 *     the raw stream finds every earlier call already queued).
 *   - arrays are column-major (Julia), element counts are size_t (8 GiB chunk = 2^31 floats).
 *   - floating-point elementwise arithmetic is IEEE round-to-nearest per operation and is
 *     NEVER contracted into FMA (Julia semantics, SURVEY Appendix A.4).
 */
#ifndef DAB200_H
#define DAB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DAB_ABI_VERSION 1

typedef struct dab_ctx dab_ctx;

/* ---- status codes ------------------------------------------------------------------ */
enum {
    DAB_OK = 0,
    DAB_ERR_CUDA = 1,         /* a CUDA runtime call failed (text in dab_last_error)            */
    DAB_ERR_ARG = 2,          /* ArgumentError: bad enum / null pointer / bad dims              */
    DAB_ERR_EMPTY = 3,        /* "reducing over an empty collection is not allowed" (max/min)   */
    DAB_ERR_DIM_MISMATCH = 4, /* DimensionMismatch (src/broadcast.jl:66, src/darray.jl:564)      */
    DAB_ERR_NCCL = 5,         /* NCCL missing or a NCCL call failed                             */
    DAB_ERR_UNSUPPORTED = 6,  /* op/dtype combination not served by a kernel: NO host fallback   */
    DAB_ERR_NVRTC = 7,        /* runtime compilation of a fused broadcast expression failed      */
    DAB_ERR_NOMEM = 8
};

/* ---- element types ----------------------------------------------------------------- */
enum { DAB_F32 = 0, DAB_F64 = 1, DAB_I32 = 2, DAB_I64 = 3, DAB_U8 = 4 /* Bool */,
       DAB_I128 = 5 /* Int128: ONLY as the value type of dab_mapreduce_expr (f widens, e.g. x -> Int128(x)^2; test/darray.jl:286-294);
                       there are no arrays of it.  Its result fills the whole 16-byte slot (two's complement, little endian). */,
       DAB_C64 = 6 /* ComplexF32 */, DAB_C128 = 7 /* ComplexF64 */, DAB_F16 = 8 /* Float16 (IEEE binary16) */ };
/* Complex element types are stored interleaved (re, im), as Julia's Complex{T}.  Entry points that accept them:
 *   dab_fill, dab_reduce / dab_reduce_host / dab_mapreduce_all / dab_reduce_result_dtype / dab_combine_ordered (see there),
 *   dab_broadcast_expr / dab_mapreduce_expr and their compile checks (argument, output and value types), dab_adjoint_box, and the
 *   byte movers that take an element size (dab_copy_box, dab_gather_box, dab_transpose_box with 8 / 16 bytes, dab_h2d, ...).
 * dab_reducedim takes them for SUM with MAP_ID only and runs it as the real SUM over (2*inner, reduce, outer) of the components (Julia's
 * complex + is componentwise); any other op or map returns DAB_ERR_UNSUPPORTED naming the dtype.  drand of a complex array calls
 * dab_rand_u01 on the real view of 2n components at global offset 2g.  Every other entry point returns DAB_ERR_UNSUPPORTED (or
 * DAB_ERR_ARG) for them, naming the dtype. */
/* Float16 (DAB_F16, 2 bytes) is accepted by:
 *   dab_fill (2-byte value), dab_rand_u01 (element g = (hash32(seed, g) >> 22) * 2^-10, Julia's rand(Float16)),
 *   dab_reduce / dab_reduce_host / dab_mapreduce_all / dab_reduce_result_dtype / dab_combine_ordered: SUM / PROD / MAX / MIN with
 *     MAP_ID, MAP_ABS, MAP_ABS2, MAP_NEG (Float16 result: fp32 over each tile step, fp64 carrier, one rounding to Float16 at the end;
 *     MAX / MIN exact), and COUNT / ANY / ALL / SUM with the predicate maps (Int64); EXTREMA returns DAB_ERR_UNSUPPORTED (extrema of
 *     Float16 data is a MIN and a MAX reduction).  dab_mapreduce_all folds Float16 results through dab_reduce + allgather + dab_combine_ordered.
 *   dab_reducedim: SUM / PROD / MAX / MIN with MAP_ID, MAP_ABS, MAP_ABS2, MAP_NEG, Float16 output.
 *   dab_broadcast_expr / dab_mapreduce_expr and their compile checks (argument, output and value types: "widen to Float32, operate,
 *     round to Float16" per operation, as Julia's Float16 methods),
 *   the byte movers with 2-byte elements (dab_copy_box, dab_gather_box, dab_transpose_box, dab_h2d, ...).
 * Every other entry point returns DAB_ERR_UNSUPPORTED (or DAB_ERR_ARG) for it, naming the dtype; the index-gather, compaction, expansion
 * and scatter kernels (dab_index_gather, dab_compact, dab_expand, dab_scatter) have no 2-byte instances. */

/* ---- reduce operators  (op argument of Base.mapreduce; src/mapreduce.jl:31) ----------- */
enum {
    DAB_SUM = 0,   /* Base.add_sum : Int32 widens to Int64, floats stay (result dtype: f32/f64/i64) */
    DAB_PROD = 1,  /* Base.mul_prod: same widening                                               */
    DAB_MAX = 2,   /* Julia max: NaN-propagating, +0.0 > -0.0                                    */
    DAB_MIN = 3,   /* Julia min                                                                  */
    DAB_ALL = 4,   /* Base._all  (src/mapreduce.jl:97-104)  result int64 0/1                     */
    DAB_ANY = 5,   /* Base._any  (src/mapreduce.jl:106-113) result int64 0/1                     */
    DAB_COUNT = 6, /* Base.count (src/mapreduce.jl:115-122) result int64                         */
    DAB_EXTREMA = 7 /* Base.extrema (src/mapreduce.jl:124-131) in ONE pass: the result slot holds (min, max) as two T (dab_reduce
                       only, MAP_ID only; the cross-worker fold takes min of mins / max of maxes)            */
};

/* ---- which argument of dab_findminmax / dab_findminmax_dim / dab_combine_findminmax ---- */
enum {
    DAB_FINDMAX = 0, /* Base.findmax: the later element wins when isless(best, x)    */
    DAB_FINDMIN = 1  /* Base.findmin: the later element wins when isgreater(best, x) */
};

/* ---- map functions f of mapreduce(f, op, A) / unary broadcast ------------------------ */
enum {
    DAB_MAP_ID = 0,
    DAB_MAP_ABS = 1,
    DAB_MAP_ABS2 = 2,
    DAB_MAP_NEG = 3,
    DAB_MAP_SQRT = 4,  /* correctly rounded */
    DAB_MAP_INV = 5,   /* 1/x correctly rounded (float only) */
    DAB_MAP_FLOOR = 6,
    DAB_MAP_CEIL = 7,
    DAB_MAP_SIGN = 8,
    /* predicates against a scalar parameter p (x -> x OP p), for all/any/count; result Bool */
    DAB_MAP_EQ = 16, DAB_MAP_NE = 17, DAB_MAP_LT = 18, DAB_MAP_LE = 19, DAB_MAP_GT = 20, DAB_MAP_GE = 21,
    DAB_MAP_ISNAN = 22, DAB_MAP_NONZERO = 23 /* identity on Bool/number -> (x != 0) */
};

/* ---- binary broadcast operators ------------------------------------------------------ */
enum {
    DAB_ADD = 0, DAB_SUB = 1, DAB_MUL = 2, DAB_DIV = 3 /* float: IEEE div; int: unsupported (Julia / gives Float64) */,
    DAB_REM = 4  /* Julia rem / % : C fmod semantics (sign of dividend); ints: truncated remainder */,
    DAB_BMAX = 5, DAB_BMIN = 6,
    DAB_MOD = 7  /* Julia mod: floored */,
    DAB_IDIV = 8 /* Julia div: truncated integer quotient (ints only) */,
    DAB_AND = 9, DAB_OR = 10, DAB_XOR = 11 /* ints only */
};

/* ==== lifecycle ======================================================================= */
int32_t dab_abi_version(void);
/* number of visible CUDA devices (0 and DAB_ERR_CUDA when there is no driver). */
int32_t dab_device_count(int32_t* count);
/* One context per worker process/device.  Replaces the implicit per-process state of a Julia
 * worker (REGISTRY, src/core.jl:1-52): creates the stream and the reduction scratch. */
int32_t dab_init(int32_t device, dab_ctx** ctx);
int32_t dab_shutdown(dab_ctx* ctx);
const char* dab_last_error(const dab_ctx* ctx); /* ctx may be NULL: last error of dab_init */
const char* dab_status_string(int32_t status);
/* remotecall_wait: block until everything queued on the ctx stream is done. */
int32_t dab_sync(dab_ctx* ctx);
int32_t dab_device_info(dab_ctx* ctx, int32_t* device, int32_t* sm_count, size_t* free_bytes, size_t* total_bytes);
/* the ctx's cudaStream_t (as void*), so a host runtime can order its own work after ours.  Queues a held-back
 * dab_affine and stops holding any back on this ctx from then on. */
int32_t dab_stream(dab_ctx* ctx, void** stream);
/* two switches; "combine_timeout_ms" = wall-clock bound of the fused combine's wait for a peer; "ew_tma" = 1 routes aligned unary elementwise launches through the TMA-staged (cp.async.bulk + mbarrier
 * ring) kernel instead of the default flat LDG/STG kernel -- identical results, measured slower (DESIGN.md section 3).  Any other key is DAB_ERR_ARG. */
int32_t dab_set_option(dab_ctx* ctx, const char* key, int64_t value);
/* number of kernels this ctx has launched so far (bench.py's gpu_launches claim). */
int32_t dab_launch_count(dab_ctx* ctx, uint64_t* launches);

/* ==== device-side timing (CUDA events on the ctx stream) ================================ */
int32_t dab_event_create(dab_ctx* ctx, void** event);
int32_t dab_event_record(dab_ctx* ctx, void* event);
int32_t dab_event_elapsed_ms(dab_ctx* ctx, void* start, void* stop, float* ms); /* syncs on stop */
int32_t dab_event_destroy(dab_ctx* ctx, void* event);

/* ==== buffers: a localpart lives in one GPU's HBM ======================================
 * Replaces Array{T}(undef, ...) on a worker (src/darray.jl:62,174,222-225).  The caller owns
 * the pointer and must dab_free it (a Julia B200Array attaches a finalizer, mirroring
 * src/darray.jl:47-49). */
int32_t dab_alloc(dab_ctx* ctx, size_t nbytes, void** dptr);
int32_t dab_free(dab_ctx* ctx, void* dptr);
/* stream-ordered temporaries (cudaMallocAsync pool; ~1 us, no synchronisation; not IPC-exportable) */
int32_t dab_alloc_async(dab_ctx* ctx, size_t nbytes, void** dptr);
int32_t dab_free_async(dab_ctx* ctx, void* dptr);
int32_t dab_host_alloc(dab_ctx* ctx, size_t nbytes, void** hptr); /* pinned staging */
int32_t dab_host_free(dab_ctx* ctx, void* hptr);
/* distribute(A) / Array(d) per chunk (src/darray.jl:544-555, 574-582): async on the ctx stream.  dab_h2d from PINNED memory is one
 * cudaMemcpyAsync; from large pageable memory it is pipelined through two pinned staging buffers (host threads fill one while the copy
 * engine drains the other) and returns once the source has been consumed, so the caller's array may be reused immediately. */
int32_t dab_h2d(dab_ctx* ctx, void* dptr, const void* hptr, size_t nbytes);
int32_t dab_d2h(dab_ctx* ctx, void* hptr, const void* dptr, size_t nbytes);
int32_t dab_d2d(dab_ctx* ctx, void* dst, const void* src, size_t nbytes);
/* 2-D strided host<->device copy of a column-major box: `cols` columns of `rows*elem` bytes
 * (distribute's A[idxs...] slicing, src/darray.jl:551).  Pitches are in bytes. */
int32_t dab_h2d_2d(dab_ctx* ctx, void* dptr, size_t dpitch, const void* hptr, size_t hpitch, size_t row_bytes, size_t cols);
int32_t dab_d2h_2d(dab_ctx* ctx, void* hptr, size_t hpitch, const void* dptr, size_t dpitch, size_t row_bytes, size_t cols);
/* fill!(localpart(A), x)  (src/darray.jl:822-827).  value points to one element of dtype. */
int32_t dab_fill(dab_ctx* ctx, int32_t dtype, void* x, size_t n, const void* value);
/* rand!(localpart(A)) (src/darray.jl:829-834) with a counter-based generator so the CPU oracle
 * can regenerate any element: x[i] = (hash32(seed, global_offset+i) >> 8) * 2^-24  in [0,1)
 * (distribution of Julia's rand(Float32)).  dtype F32 or F64. */
int32_t dab_rand_u01(dab_ctx* ctx, int32_t dtype, void* x, size_t n, uint64_t seed, uint64_t global_offset);

/* ==== elementwise kernels K1-K3 (HBM-bound, 8 B/element) ===============================
 * Replace the Base loop run on each localpart by
 *   copyto!(localpart(dest), lbc)            src/broadcast.jl:80   (y .= a .* x .+ b)
 *   copy(lbc)                                src/broadcast.jl:96   (map / allocating broadcast)
 *   map!(f, localpart(dest), makelocal(...)) src/mapreduce.jl:8    (map!(x->2x+1, d, d))
 * y may alias x exactly (in place).  a, b, s point to one host scalar of dtype. */
int32_t dab_affine(dab_ctx* ctx, int32_t dtype, void* y, const void* x, const void* a, const void* b, size_t n);
/* y = fn(x), fn from the DAB_MAP_* enum (non-predicate entries). */
int32_t dab_unary(dab_ctx* ctx, int32_t dtype, int32_t fn, void* y, const void* x, size_t n);
/* z = x OP y  (same-shape DArray .op DArray; also map_localparts binary ops src/mapreduce.jl:134-189). */
int32_t dab_binary(dab_ctx* ctx, int32_t dtype, int32_t op, void* z, const void* x, const void* y, size_t n);
/* z = x OP s (scalar_left == 0) or z = s OP x (scalar_left != 0). */
int32_t dab_binary_scalar(dab_ctx* ctx, int32_t dtype, int32_t op, void* z, const void* x, const void* s,
                          int32_t scalar_left, size_t n);
/* General fused broadcast  dest .= f.(args...)  for an arbitrary expression tree, compiled at run
 * time with NVRTC for sm_90a (what Julia's JIT does for a Broadcasted, src/broadcast.jl:65-85).
 * `expr` is C source for ONE element in terms of a0..a{nargs-1} (already converted to their
 * dtypes) and must yield a value of out_dtype, e.g. "a0 - a1 * sinf(a2)".  Each arg k is either
 * a device array (arg_ptrs[k] != NULL) indexed through arg_strides[k*4 .. k*4+3] (0 for an extruded
 * / size-1 dim, src/broadcast.jl:112-113) over the destination box shape[0..3] (column-major,
 * unused dims = 1), or a scalar passed by value through arg_scalars[k] (8 bytes each).
 * Compiled kernels are cached per (expr, dtypes, arg kinds). */
int32_t dab_broadcast_expr(dab_ctx* ctx, const char* expr, int32_t out_dtype, void* out, const size_t shape[4],
                           const size_t out_strides[4], int32_t nargs, const int32_t* arg_dtypes,
                           const void* const* arg_ptrs, const size_t* arg_strides, const uint64_t* arg_scalars);

/* Diagnostic, needs no GPU: generate + NVRTC-compile the kernels dab_broadcast_expr would use for this expression and
 * report the sm_90a cubin size (arg_is_array[k] != 0: array argument, else by-value scalar). */
int32_t dab_jit_compile_check(const char* expr, int32_t out_dtype, int32_t nargs, const int32_t* arg_dtypes,
                              const int32_t* arg_is_array, size_t* cubin_bytes);

/* Fused map + reduce of an arbitrary traced expression over one localpart, ONE pass over HBM:  mapreduce(f, op, args...)
 * (reference src/mapreduce.jl:31 with a general closure f; dot(x, y) = mapreduce(*, +, x, y); d == a via all(x .== y)).
 * expr / args as in dab_broadcast_expr but all array arguments are dense with n elements (linear indexing); val_dtype is the
 * type of the expression's value.  The 16-byte result slot at out_dev has the layout of dab_reduce (val_dtype DAB_I128, ops SUM / PROD /
 * MAX / MIN: the slot IS the Int128 result; wrap-around arithmetic like Julia's).  NVRTC-compiled, cached. */
int32_t dab_mapreduce_expr(dab_ctx* ctx, const char* expr, int32_t val_dtype, int32_t op, size_t n, int32_t nargs, const int32_t* arg_dtypes,
                           const void* const* arg_ptrs, const uint64_t* arg_scalars, void* out_dev);
int32_t dab_jit_compile_check_reduce(const char* expr, int32_t val_dtype, int32_t op, int32_t nargs, const int32_t* arg_dtypes,
                                     const int32_t* arg_is_array, size_t* cubin_bytes);
/* Diagnostic (no GPU, no NVRTC): the generated CUDA source -- kind 0 dab_broadcast_expr's kernels (dtype = output type), kind 1
 * dab_mapreduce_expr's (dtype = value type, op).  At most cap bytes go to buf, the full length to *len. */
int32_t dab_jit_source(int32_t kind, const char* expr, int32_t dtype, int32_t op, int32_t nargs, const int32_t* arg_dtypes,
                       const int32_t* arg_is_array, char* buf, size_t cap, size_t* len);

/* ==== whole-chunk reductions K4 / K7 (HBM-bound, 4 B/element) ==========================
 * Replace mapreduce(f, op, localpart(d)) / reduce(f, localpart(d)) run per worker at
 * src/mapreduce.jl:23,31 and all/any/count/extrema at :100,109,118,127.
 * The chunk result (ONE value of the result dtype: f32/f64 for float SUM/PROD, int64 for integer
 * SUM/PROD and ALL/ANY/COUNT, T for MAX/MIN) is written to out_dev, which must have room for 16 bytes:
 * [0,8) the result in its result dtype, [8,16) the wide carrier (fp64 for float SUM/PROD, else a copy).
 * Float sums are accumulated in fp32 over <=16-element groups and carried in fp64 (more accurate
 * than Base's pairwise fp32; within 1e-6 rel of it -- SURVEY 8c).  map_param: host scalar of dtype for
 * predicate maps, else NULL.  n == 0: SUM->0, PROD->1, ALL->1, ANY/COUNT->0, MAX/MIN -> DAB_ERR_EMPTY. */
int32_t dab_reduce(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* map_param, const void* x, size_t n,
                   void* out_dev);
/* Complex dtypes (C64 / C128; x 8- resp. 16-byte aligned):
 *   SUM / PROD with MAP_ID or MAP_NEG -> complex result: it fills [0, 2*sizeof(T)) of the slot, the rest is zero (no separate carrier).
 *     Sums add each component in T over a 16-byte tile step and carry them in fp64 (Julia's complex + is componentwise); products
 *     multiply (ac - bd, ad + bc) with every operation rounded separately, in a complex fp64 carrier, rounded once to T.
 *   SUM / MAX / MIN with MAP_ABS2 (re*re + im*im) or MAP_ABS (hypot) -> real result of the component type, laid out as for that type.
 *   COUNT / ANY / ALL with MAP_NONZERO or MAP_ISNAN (either component NaN) -> Int64.
 *   Anything else (MAX / MIN / EXTREMA with MAP_ID, PROD of a map, other maps) -> DAB_ERR_UNSUPPORTED. */
/* Same, then copies the 16-byte result slot to out_host and syncs (== remotecall_fetch, src/mapreduce.jl:31). */
int32_t dab_reduce_host(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* map_param, const void* x,
                        size_t n, void* out_host);
/* result dtype of dab_reduce for (dtype, op, map). */
int32_t dab_reduce_result_dtype(int32_t dtype, int32_t op, int32_t map, int32_t* out_dtype);
/* Caller-side combine  reduce(op, results)  (src/mapreduce.jl:26,34): P < 16 so a plain LEFT FOLD in
 * procs(d) order, in the result dtype (Float32 partials fold in Float32; ComplexF32 partials fold in Float32 arithmetic,
 * componentwise for SUM and as (ac - bd, ad + bc) for PROD).  Host arrays. */
int32_t dab_combine_ordered(int32_t result_dtype, int32_t op, const void* partials_host, size_t p, void* out_host);

/* ==== dimensional reduction K5 / K6 =====================================================
 * Replaces mapreduce(f, op, localpart(A), dims=region) (src/mapreduce.jl:64, phase 1) and
 * Base.mapreducedim!(f, op, localpart(R), B) (src/mapreduce.jl:77, phase 2) on the chunk collapsed to
 * the column-major shape (inner, reduce, outer): out[i + inner*o] (op)= x[i + inner*(r + reduce*o)].
 * accumulate == 0: out is overwritten with the reduction (SUM/PROD seeded with 0/1, MAX/MIN with
 * the first element); accumulate != 0: the reduction is combined ONTO the existing out
 * (how init= and the between-phase enter, SURVEY Appendix A.3).  For float SUM / PROD the combine
 * rounds op(out, S) ONCE to the output type: S, the reduction, stays in its fp64 carrier until then,
 * on every launch path.  Output dtype follows dab_reduce_result_dtype. */
int32_t dab_reducedim(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* x, size_t inner, size_t reduce,
                      size_t outer, void* out, int32_t accumulate);

/* ==== findmax / findmin K20 ================================================================
 * Replace Base's findmax(f, A) / findmin(f, A) (_findmax) and findminmax!(f, op, Rval, Rind, A) (the dims form) on one chunk.  The winner
 * is the element with the largest order key, then the smallest linear index: Julia's isless order of f(x) for DAB_FINDMAX, reversed for
 * DAB_FINDMIN, with every NaN on top for both (NaN wins, the first NaN is kept; findmax prefers +0.0, findmin -0.0; ties keep the earlier
 * index).  dtype: F32 F64 I32 I64, and U8 holding Bool (0 / 1).  map: MAP_ID, MAP_ABS, MAP_ABS2 (Int32 abs / abs2 wrap as in Julia; both
 * are the identity on Bool).  Complex dtypes and other maps -> DAB_ERR_UNSUPPORTED, a bad `which` -> DAB_ERR_ARG, before the context is
 * touched.  x must be aligned to its element size; any 16-byte phase is served.
 *
 * dab_findminmax: out_dev gets 16 bytes: [0, 8) f(x[i]) as T (zero-padded; the element itself, so a NaN keeps its payload), [8, 16) i,
 * the 0-based chunk-local linear index, as Int64.  map_param: unused (NULL).  n == 0 -> DAB_ERR_EMPTY. */
int32_t dab_findminmax(dab_ctx* ctx, int32_t dtype, int32_t which, int32_t map, const void* map_param, const void* x, size_t n,
                       void* out_dev);
/* dab_findminmax_dim: x collapsed to (inner, reduce, outer) as in dab_reducedim; out_vals[i + inner*o] (T) and out_idx[i + inner*o]
 * (Int64) are the winner of x[i + inner*(r + reduce*o)], r = 0 .. reduce-1.  out_idx is the 1-based GLOBAL linear index of the winner:
 * its chunk-local position unravelled in chunk_dims[0..nd), shifted by the 0-based offsets[], ravelled in global_dims[] (nd <= 8;
 * nd == 0: the position itself plus one).  idx_in (optional, MAP_ID only): an Int64 array shaped like x holding each value's 1-based
 * global index already; the winner's index is then taken from it and compared as such (a second reduced run, the fold of exchanged
 * slabs).  inner * outer == 0: nothing to do; reduce == 0 -> DAB_ERR_EMPTY. */
int32_t dab_findminmax_dim(dab_ctx* ctx, int32_t dtype, int32_t which, int32_t map, const void* x, const int64_t* idx_in, size_t inner,
                           size_t reduce, size_t outer, int32_t nd, const int64_t* chunk_dims, const int64_t* offsets,
                           const int64_t* global_dims, void* out_vals, int64_t* out_idx);
/* Host-only: the winner of `count` 16-byte records (value as T in [0, 8), Int64 index in [8, 16), any one index convention) under the
 * order above, copied to out (16 bytes).  Lets the chunk results of dab_findminmax, made global, be folded in any order. */
int32_t dab_combine_findminmax(int32_t dtype, int32_t which, const void* records, size_t count, void* out);

/* ==== scans K17: accumulate! / cumsum! / cumprod! =========================================
 * Replaces Base's accumulate!(op, B, A; dims, init) (base/accumulate.jl: _accumulate!, accumulate_pairwise / the per-fibre loop
 * with reduce_first) on one chunk collapsed to the column-major shape (inner, len, outer) around dims:
 *   y[i + inner*(r + len*o)] = c[k] (op) x[i + inner*(len*o)] (op) ... (op) x[i + inner*(r + len*o)],  k = i + inner*o,
 * where c is the carry slab: inner*outer values in the CARRIER type (below), the exclusive prefix contributed by init and by earlier
 * chunks along dims.  carry == NULL: no prefix, the first output of every fibre is reduce_first(op, x) (converted to out_dtype).
 * Served (in_dtype, op, out_dtype), op in SUM PROD MAX MIN (Julia's + * max min: NaN-propagating, max(-0.0, 0.0) = 0.0):
 *   F32 / F64 / I64 -> the same type;  I32: SUM / PROD -> I64 (cumsum / cumprod: add_sum / mul_prod widen) or I32 (accumulate(+ / *):
 *   wraps at 32 bits), MAX / MIN -> I32;  U8 (Bool): SUM -> I64, PROD -> U8 (AND), MAX / MIN -> U8 (OR / AND).
 *   Anything else returns DAB_ERR_UNSUPPORTED.
 * Carriers: F64 for float SUM / PROD (each output rounded once from the fp64 prefix), I64 for integer and Bool SUM / PROD (an I32
 * result keeps the low 32 bits), the element type for MAX / MIN (dab_scan_carrier_dtype).  Float results are not bit-identical to
 * Julia's sequential fold: the parallel order differs, and Float32 prefixes run in fp64 (DESIGN.md section 7).
 * inner == 1: one single-pass kernel with a decoupled look-back across tiles; inner > 1: threads along inner walk len, split into
 * segments (one extra read) when inner*outer cannot fill the GPU.  The 16-byte loads / stores need x / y aligned to 16 bytes (the host
 * runtime's chunks are 256-byte aligned); a misaligned base is served for the whole call with coalesced element loads / stores -- the
 * same results, without a head peel.  x == y (in place) is allowed when in and out elements have the same
 * size; other overlaps are not.  Asynchronous on the ctx stream. */
int32_t dab_scan(dab_ctx* ctx, int32_t in_dtype, int32_t op, int32_t out_dtype, const void* x, size_t inner, size_t len, size_t outer,
                 const void* carry, void* y);
/* totals[k] = x[i + inner*(len*o)] (op) ... (op) x[i + inner*(len - 1 + len*o)] in the carrier type, k = i + inner*o (the identity of op
 * when len == 0): the chunk totals that the host folds, in grid order along dims, into the carries of the later chunks.  Same
 * (in_dtype, op, out_dtype) table and kernels as dab_scan, storing only the totals. */
int32_t dab_scan_totals(dab_ctx* ctx, int32_t in_dtype, int32_t op, int32_t out_dtype, const void* x, size_t inner, size_t len, size_t outer,
                        void* totals);
/* carrier dtype of dab_scan for (in_dtype, op, out_dtype); DAB_ERR_UNSUPPORTED when the triple is not served.  Host only. */
int32_t dab_scan_carrier_dtype(int32_t in_dtype, int32_t op, int32_t out_dtype, int32_t* carrier_dtype);

/* ==== slab / halo copy K8 ===============================================================
 * Replaces the owner-side  localpart(d)[idxs...]  + serialise + TCP + a[idxs...] = ...  of
 * setindex!(::Array, ::SubDArray, ...) (src/darray.jl:798-820), chunk() (:458) and the non-local
 * branch of makelocal (:361-366).  Copies a box of `extent` elements (up to 4 dims, column-major)
 * from src (array shape src_shape, box origin src_off, 0-based) to dst.  src may be a pointer into
 * ANOTHER GPU's memory (peer-enabled in-process, or opened with dab_ipc_open): the copy kernel
 * then pulls over NVLink with 16-byte loads -- one-sided, like the reference's pull-style read. */
int32_t dab_copy_box(dab_ctx* ctx, int32_t elem_bytes, void* dst, const size_t dst_shape[4], const size_t dst_off[4],
                     const void* src, const size_t src_shape[4], const size_t src_off[4], const size_t extent[4]);

/* Strided and vector-indexed views: the piece of Array(d[I...]) held by one chunk when some index is a StepRange or a Vector{Int}
 * (src/darray.jl:661, 798-820; indexin_mask / restrict_indices :706-781).  ndim <= 8.  Coordinate t of dimension k contributes
 * t * dst_strides[k] (resp. src_strides[k], may be negative) ELEMENTS to the destination (source) offset, or, when dst_index[k]
 * (src_index[k]) is non-NULL, the value table[k][t] of a device array of int64 element offsets.  dst / src point at the element of
 * coordinate 0; src may be a peer mapping.  dst_index / src_index may be NULL (all affine). */
int32_t dab_gather_box(dab_ctx* ctx, int32_t elem_bytes, int32_t ndim, void* dst, const long long* dst_strides, const void* const* dst_index,
                       const void* src, const long long* src_strides, const void* const* src_index, const size_t* extent);

/* ==== dimension permutation K28 (row f18) ===================================================
 * dst[sum_k t_k * dst_strides[k]] = src[sum_k t_k * src_strides[k]] for every coordinate t < extent: one piece of permutedims(A, perm)
 * / permutedims!(dest, src, perm), which Base computes with one scalar getindex (one remotecall_fetch) per element on a DArray.  This
 * is the affine part of dab_gather_box's contract, restricted to boxes where dimension 0 is contiguous in the destination
 * (dst_strides[0] == 1) and exactly one other dimension q is contiguous in the source (src_strides[q] == 1); it replaces
 * dab_gather_box on those pieces, whose warps would read or write with a stride.  Each CTA moves one tile of the (0, q) plane through
 * shared memory, the other dimensions being a batch; 16-byte global accesses on both sides when dst, src, the strides outside the
 * plane and both plane extents allow it.  ndim 2..8, elem_bytes 1, 2, 4, 8 or 16 (bytes are moved: NaN payloads and -0.0 kept);
 * strides in elements, may be negative.  src may be a peer mapping.  Anything else returns DAB_ERR_ARG and touches nothing; a zero
 * extent launches nothing.  One launch per call, asynchronous on the ctx stream. */
int32_t dab_permute_box(dab_ctx* ctx, int32_t elem_bytes, int32_t ndim, void* dst, const long long* dst_strides, const void* src,
                        const long long* src_strides, const size_t* extent);

/* ==== indexed gather K22 (row f12) ==========================================================
 * out[k] = d[idx[k]] for k < n: one localpart of R = d[I::DArray{<:Integer}], which Base's generic getindex computes as
 * similar(d, axes(I)) (src/darray.jl:238) filled by scalar reads.  idx holds the matching block of I: 1-based column-major LINEAR
 * indices into the whole source d (Julia's A[I::AbstractArray{<:Integer}]); idx_dtype DAB_I32 (widened to 64 bits in the kernel)
 * or DAB_I64.  Duplicates are allowed.  The source is described by its ndim (1..8) dims, its grid (chunks per dim) and, per dim,
 * grid[k] + 1 cuts (0-based first element of each chunk along the dim, then dims[k]; empty chunks repeat a cut), concatenated dim
 * by dim, and one pointer per chunk in column-major grid order: local or a CUDA-IPC peer mapping, NULL allowed for an empty chunk.
 * At most 1024 chunks (otherwise DAB_ERR_UNSUPPORTED); the table travels by value in the kernel's parameter block.  elem_bytes
 * 1, 4, 8 or 16: the kernel moves bytes, so NaN payloads and -0.0 are kept.  out aligned to elem_bytes, idx to its element size;
 * 16-byte aligned idx and out take the 16-byte index loads.  Bounds: an index outside [1, prod(dims)] writes nothing for that
 * element and atomicMin's its position k into *bad_pos (device, 8 bytes), which the caller initialises to ULLONG_MAX.  n == 0
 * launches nothing.  Asynchronous on the ctx stream. */
int32_t dab_index_gather(dab_ctx* ctx, int32_t elem_bytes, void* out, const void* idx, int32_t idx_dtype, size_t n, int32_t ndim,
                         const size_t* dims, const int32_t* grid, const size_t* cuts, const void* const* chunk_ptrs,
                         unsigned long long* bad_pos);

/* ==== stream compaction K23 (row f13) ========================================================
 * The kernels of d[mask::DArray{Bool}], findall(mask) and filter(f, d), which Base computes by scalar iteration.  One call serves
 * one chunk, cut into `runs` RUNS of run_len elements that lie back to back in the chunk's storage and are each contiguous in the
 * global column-major order (the host derives them from the layout: DESIGN.md section 3.10).  Each run is cut into
 * tiles_per_run = ceil(run_len / DAB_COMPACT_TILE) tiles; tile b = r * tiles_per_run + t covers chunk elements
 * [r * run_len + t * DAB_COMPACT_TILE, r * run_len + min((t + 1) * DAB_COMPACT_TILE, run_len)).  A mask byte is true when nonzero.
 * The mask may have any alignment (16-byte loads where a tile starts 16-byte aligned).  Asynchronous on the ctx stream;
 * run_len == 0 or runs == 0 launches nothing.  More than 2^31 - 1 tiles: DAB_ERR_UNSUPPORTED. */
#define DAB_COMPACT_TILE 4096
#define DAB_COMPACT_INDEX 0
/* counts[b] (Int32) = the number of true bytes of mask tile b. */
int32_t dab_compact_count(dab_ctx* ctx, const void* mask, size_t run_len, size_t runs, int32_t* counts);
/* Writes the selected elements of the chunk, in order, to a 1-D output of nchunks (1..1024) chunks: the element at run position i
 * of run r that is the p-th true of its run goes to output position run_info[2r] + p.  tile_incl: the Int64 inclusive scan of
 * counts along each run (dab_scan DAB_I32 -> DAB_I64, SUM, inner 1, len tiles_per_run, outer runs).  The output is described by
 * nchunks + 1 cuts (0-based first position of each chunk, then its length; empty chunks repeat a cut) and one pointer per chunk,
 * local or a CUDA-IPC peer mapping (NULL allowed for an empty chunk), passed by value.  elem_bytes 1, 4, 8 or 16: src[element] is
 * copied as bytes (NaN payloads and -0.0 kept); elem_bytes == DAB_COMPACT_INDEX: the Int64 run_info[2r + 1] + i + 1 is written
 * (run_info[2r + 1] is the 0-based global linear index of the run's first element; src unused).  Positions at or past the output
 * length are not written. */
int32_t dab_compact(dab_ctx* ctx, int32_t elem_bytes, const void* mask, const void* src, size_t run_len, size_t runs, const int64_t* tile_incl,
                    const int64_t* run_info, int32_t nchunks, const size_t* cuts, void* const* chunk_ptrs);

/* ==== indexed scatter K24 (row f14) =========================================================
 * d[I[k]] = v[k]: one block of I::DArray{<:Integer} (1-based column-major LINEAR indices into the whole destination d, idx_dtype
 * DAB_I32 or DAB_I64) per call, the inverse of K22.  The destination is described exactly as dab_index_gather's source (ndim, dims,
 * grid, cuts, one pointer per chunk, local or a CUDA-IPC peer mapping, at most 1024 chunks); NaN payloads and -0.0 are stored as
 * bytes.  Julia's setindex! is sequential, so the host runs, over every block of I, first dab_scatter_check, then (when a duplicate
 * was flagged) dab_scatter_winners, then dab_scatter.  n == 0 launches nothing.  Asynchronous on the ctx stream. */
/* Bounds and duplicates.  bitmap_ptrs: one zeroed bitmap of ceil(chunk length / 32) uint32 words per chunk of d (same table shape as
 * chunk_ptrs, 4-byte aligned).  An index outside [1, prod(dims)] atomicMin's its block position into status[0] (initialise it to
 * ULLONG_MAX); every valid index sets the bit of its element (atomicOr) and, when the bit was set already, sets status[1] to 1
 * (initialise it to 0).  d itself is not read or written. */
int32_t dab_scatter_check(dab_ctx* ctx, const void* idx, int32_t idx_dtype, size_t n, int32_t ndim, const size_t* dims, const int32_t* grid,
                          const size_t* cuts, void* const* bitmap_ptrs, unsigned long long* status);
/* The last occurrence of every destination: atomicMax of p + 1 into the winner table at the element of idx[k], with p the 0-based
 * global column-major position of block element k in I: the block is a stack of runs of run_len elements, contiguous in I's global
 * order, run r starting at run_lin[r] (Int64, device).  win_ptrs: one zeroed table of win_bytes (4, or 8 when length(I) >= 2^32) per
 * element of each chunk of d.  Out-of-range indices are skipped. */
int32_t dab_scatter_winners(dab_ctx* ctx, const void* idx, int32_t idx_dtype, size_t n, size_t run_len, const int64_t* run_lin, int32_t win_bytes,
                            int32_t ndim, const size_t* dims, const int32_t* grid, const size_t* cuts, void* const* win_ptrs);
/* The stores: the element of idx[k] takes src[k] (src: the block's values, aligned to elem_bytes 1, 4, 8 or 16) or, when src is NULL,
 * the elem_bytes at the host pointer `scalar`.  win_bytes 0: every valid index stores (the indices are unique); 4 or 8: only the index
 * whose p + 1 (as in dab_scatter_winners, with the same run table) equals its element's winner entry.  Out-of-range indices store
 * nothing. */
int32_t dab_scatter(dab_ctx* ctx, int32_t elem_bytes, const void* idx, int32_t idx_dtype, size_t n, const void* src, const void* scalar,
                    size_t run_len, const int64_t* run_lin, int32_t win_bytes, int32_t ndim, const size_t* dims, const int32_t* grid,
                    const size_t* cuts, void* const* chunk_ptrs, void* const* win_ptrs);

/* ==== masked expansion K25 (row f14) =========================================================
 * d[mask] = v, the inverse of dab_compact on the same tile table and plan (run_len, runs, tile_incl, run_info as there): the element
 * of the chunk dst at run position i of run r that is the p-th true of its run takes v[run_info[2r] + p], read through the 1-D value
 * table (nchunks 1..1024, nchunks + 1 cuts, one pointer per chunk, local or a CUDA-IPC peer mapping).  Positions at or past the
 * values' length are not read.  scalar != NULL: every selected element takes the elem_bytes at the host pointer scalar, and tile_incl,
 * run_info and the table are not used (NULL allowed).  elem_bytes 1, 4, 8 or 16, moved as bytes.  run_len == 0 or runs == 0 launches
 * nothing.  Asynchronous on the ctx stream. */
int32_t dab_expand(dab_ctx* ctx, int32_t elem_bytes, const void* mask, void* dst, size_t run_len, size_t runs, const int64_t* tile_incl,
                   const int64_t* run_info, int32_t nchunks, const size_t* cuts, const void* const* chunk_ptrs, const void* scalar);

/* ==== Level-2 linear algebra K9 (widening row f4; HBM-bound) ==============================
 * r = op(A) * x on ONE column-major chunk A (m x n, leading dimension m): trans = 0 -> r[m] = A x[n];
 * trans = 1 -> r[n] = A' x[m].  Replaces  localpart(A)*convert(localtype(x), xj)  (src/linalg.jl:95-97)
 * and  localpart(A)'*...  (:141) inside mul!(y::DVector, A::DMatrix, x, a, b); the tile results are then
 * combined into y by the caller exactly as the reference does (scale y by b, add a*R[i,j] in j order,
 * :101-117).  Float products accumulate in fp64 and round once; Int32/Int64 wrap.  dtypes: F32 F64 I32 I64. */
int32_t dab_gemv(dab_ctx* ctx, int32_t dtype, int32_t trans, const void* A, size_t m, size_t n, const void* x, void* r);

/* ==== sparse tile products K18 / K19 (row f9: SparseMatrixCSC chunks) ======================
 * K18.  out[r] = (((0 + val[p0]*x[idx[p0]]) + val[p0+1]*x[idx[p0+1]]) + ...) over p in [ptr[r], ptr[r+1]), r < nrows, in storage order,
 * in the element type, every product and add rounded on its own; Int32 / Int64 wrap.  Replaces  localpart(A)*xj  and  localpart(A)'*xj
 * (src/linalg.jl:95-97, 141) for a SparseMatrixCSC chunk, i.e. SparseArrays' _spmatmul! / _At_or_Ac_mul_B! loops: on the CSC arrays
 * (ptr = colptr, idx = rowval) it is A'*x; on the row-major copy of dab_csc_to_csr it is A*x.  ptr: nrows + 1 Int64 (0-based offsets),
 * idx: Int32, val and x: dtype; nnz = ptr[nrows] - ptr[0], below 2^32 (it chooses the lanes per row).  out is overwritten; an empty row
 * gives 0.  dtypes F32 F64 I32 I64.  Asynchronous on the ctx stream. */
int32_t dab_spmv(dab_ctx* ctx, int32_t dtype, size_t nrows, size_t nnz, const void* ptr, const void* idx, const void* val, const void* x,
                 void* out);
/* K19.  Row-major copy of one m x n CSC chunk (colptr: n + 1 Int64, rowval: Int32 sorted within each column, nzval: nnz of dtype) into
 * rowptr (m + 1 Int64), colidx (Int32) and val, rows ascending and columns ascending within each row.  Packs row << 32 | k per stored
 * entry and sorts the words with dab_sort (K11).  m, n <= 2^31 - 1 and nnz < 2^32 - 4096, otherwise DAB_ERR_UNSUPPORTED.  Sort scratch
 * (16 bytes per entry) is allocated and freed stream-ordered.  dtypes F32 F64 I32 I64.  Asynchronous on the ctx stream. */
int32_t dab_csc_to_csr(dab_ctx* ctx, int32_t dtype, size_t m, size_t n, size_t nnz, const void* colptr, const void* rowval, const void* nzval,
                       void* rowptr, void* colidx, void* val);

/* ==== Level-3 tile product K12 (widening row f4; the one contraction on the path: tensor-core roofline) =====================
 * R[m x n] (ldc) = op(A) * B on column-major operands of ONE worker: transA = 0 -> A is m x k (lda); transA = 1 -> op(A) = A^T with A
 * stored k x m (lda); B is k x n (ldb).  Replaces  localpart(A) * convert(localtype(B), Bjk)  and the transpose / adjoint forms of
 * _matmatmul! (src/linalg.jl:218-226); the caller scales C by beta and adds alpha * R per tile exactly as the reference (:232-252).
 * Float32 with 16-byte aligned bases and leading dimensions: TMA-fed wgmma (3xTF32 error-compensated, register partials drained
 * every 64 k for fp32 round-to-nearest accumulation); otherwise and for Float64 / Int32 / Int64: shared-memory tiled FMA kernel
 * (integers wrap like Julia's).  n == 1 with a dense A (lda == its row count) IS a matrix-vector product and is served by K9
 * (dab_gemv: one read of A at the HBM roofline).  R is overwritten. */
int32_t dab_gemm(dab_ctx* ctx, int32_t dtype, int32_t transA, size_t m, size_t n, size_t k, const void* A, size_t lda, const void* B,
                 size_t ldb, void* C, size_t ldc);

/* dst[j + i*dst_ld] = src[i + j*src_ld] for i < rows, j < cols (both column-major): the per-piece body of
 * copy(::Transpose/Adjoint{T,<:DArray{T,2}}) (src/linalg.jl:1-17: transpose!(lp, Array(D[reverse(I)...]))).
 * src may be a PEER pointer: rows are pulled coalesced over NVLink and written coalesced locally through a
 * shared-memory tile, so the fetched block is never materialised untransposed.  elem_bytes in {1,2,4,8,16}. */
int32_t dab_transpose_box(dab_ctx* ctx, int32_t elem_bytes, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows,
                          size_t cols);
/* dst[j + i*dst_ld] = conj(src[i + j*src_ld]): the per-piece body of copy(::Adjoint{<:Complex,<:DArray}) -- dab_transpose_box's tile
 * scheme with the imaginary component negated on the way through (sign bit flipped: NaN payloads kept).  src may be a PEER pointer.
 * dtype DAB_C64 or DAB_C128 (the adjoint of a real matrix is its transpose: dab_transpose_box). */
int32_t dab_adjoint_box(dab_ctx* ctx, int32_t dtype, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows, size_t cols);

/* ==== sort K11 (widening row f4; HBM-bound integer work) ===================================
 * out = sort(in) for one chunk: the  sort(lp; kwargs...)  of sample_n_setup_ref (src/sort.jl:8) and the
 * sort!(lp_sorting)  of scatter_n_sort_localparts (:61).  Ascending in Julia's isless order (-0.0 < 0.0,
 * NaNs last, bit patterns preserved).  LSD radix sort, 8-bit digits; passes whose digit is constant over
 * the chunk are skipped.  tmp: scratch of n elements, distinct from in/out (may be NULL when n <= 1024 and
 * in != out); in == out sorts in place.  Asynchronous on the ctx stream (histograms, pass selection and buffer
 * ping-pong are planned on the device).  dtypes: F32 F64 I32 I64. */
int32_t dab_sort(dab_ctx* ctx, int32_t dtype, const void* in, void* out, void* tmp, size_t n);

/* vals_out = vals reordered by the STABLE ascending order of keys: the  sort(lp; by = f)  /  sort!(lp_sorting; by = f)  of the
 * samplesort with a key function (src/sort.jl:8, 22, 61; `by` is accepted at :111) once the caller has evaluated keys = f.(lp)
 * (dab_broadcast_expr).  Key order is Julia's isless (-0.0 < 0.0; NaN keys last and equal to each other), elements with equal keys
 * keep their input order (Julia's default algorithm for a keyed sort is stable).  A 32-bit radix key and the element's position are
 * packed into one Int64 word per element and sorted by dab_sort (two rounds, least-significant half first, for 64-bit keys); the
 * low halves of the sorted words are the permutation applied to vals.  key dtypes F32 F64 I32 I64; val_bytes 4 or 8; n < 2^32;
 * vals_out must not alias vals.  scratch: device memory of at least dab_sort_by_key_scratch_bytes() bytes, 16-byte aligned.
 * Asynchronous on the ctx stream. */
int32_t dab_sort_by_key(dab_ctx* ctx, int32_t key_dtype, const void* keys, int32_t val_bytes, const void* vals, void* vals_out,
                        void* scratch, size_t scratch_bytes, size_t n);
int32_t dab_sort_by_key_scratch_bytes(int32_t key_dtype, size_t n, size_t* bytes);

/* ==== pair sort K21 (row f11) ================================================================
 * keys_out / vals_out = keys / vals in the stable isless order of keys (all NaNs equal); vals == NULL means vals[i] = base + i.
 * The per-chunk step of sortperm: with vals == NULL and base = the chunk's first global index, vals_out is the chunk's permutation.
 * Key order is Julia's isless (-0.0 < 0.0, NaNs last); every NaN key is equal to every other, so elements with equal keys -- NaNs
 * included -- keep their input order.  K11's onesweep passes with a 4-byte position carried beside every key; the last pass writes
 * the Int64 value (base + position, or vals[position]).  The sorted keys are bit-identical to dab_sort's except that every NaN comes
 * out as one canonical NaN.  key dtypes F32 F64 I32 I64; n < 2^32 - 4096 (otherwise DAB_ERR_UNSUPPORTED).  Aliasing: keys_out may
 * equal keys (in-place); vals_out must not overlap vals, keys or keys_out; no other overlap is allowed.  scratch: device memory of
 * at least dab_sort_pairs_scratch_bytes() bytes, 16-byte aligned.  Asynchronous on the ctx stream (the pass plan is made on the
 * device, as in dab_sort). */
int32_t dab_sort_pairs_scratch_bytes(int32_t key_dtype, size_t n, size_t* bytes);
int32_t dab_sort_pairs(dab_ctx* ctx, int32_t key_dtype, const void* keys, void* keys_out, const int64_t* vals, int64_t base,
                       int64_t* vals_out, void* scratch, size_t scratch_bytes, size_t n);

/* Split points of a sorted chunk for the boundaries of the samplesort (src/sort.jl:28-40): for each of the
 * nb (<= 256) host values bounds[i] (dtype elements), counts_host[i] = the number of leading elements the
 * reference's scan would pass before the first x > bounds[i] had it started at element 1 -- the count of
 * non-NaN elements <= bounds[i], or n when nothing exceeds the bound (NaNs compare false and stay).
 * Synchronous (returns with counts_host filled). */
int32_t dab_sorted_split(dab_ctx* ctx, int32_t dtype, const void* sorted, size_t n, const void* bounds_host, int32_t nb,
                         unsigned long long* counts_host);

/* ==== slice functions of mapslices(f, D; dims) (src/mapreduce.jl:191-208) =================
 * The  mapslices(f, localpart(y), dims=z)  run on every worker (:205) for the f that need a kernel of their own. */

/* Longest fibre dab_sort_slices sorts in shared memory; longer fibres go through K11 (dab_sort) one by one. */
#define DAB_SORT_SLICES_SMEM_LEN 8192
/* out[fibre] = sort(in[fibre]) for every fibre x[i + inner*(r + len*o)], r < len, of the column-major (inner, len, outer) box, i < inner,
 * o < outer: mapslices(sort, lp, dims=d) with the chunk collapsed around dimension d.  Julia's isless order (SortKey<T>, as K11); every
 * output fibre is bit-identical to dab_sort of that fibre (NaNs included: the key encoding is a bijection).  in == out sorts in place;
 * other overlaps are not allowed.  Scratch of the long-fibre path comes from the ctx block cache.  dtypes: F32 F64 I32 I64. */
int32_t dab_sort_slices(dab_ctx* ctx, int32_t dtype, const void* in, void* out, size_t inner, size_t len, size_t outer);

/* ==== sortperm along a dimension K26 (row f15) ============================================
 * The  sortperm(A; dims=dim)  of one chunk in which dimension dim (1-based) is whole.  The chunk (ndim <= 8 column-major dims chunk_dims,
 * first global index chunk_lo[k], 0-based, in an array of global_dims) is collapsed to (inner, len, outer) around dim.  For every fibre
 * (i, o) and rank r < len:  perm[i + inner*(r + len*o)] = the 1-based global column-major linear index of the fibre element of rank r in
 * the stable isless order of keys (-0.0 < 0.0; NaNs last, equal to each other, so they keep their input order) -- Julia's
 * sortperm(A; dims) entries, LinearIndices(A).  With vals / vals_out (both or neither; val_bytes 4 or 8) that element's value is moved
 * to the same place of vals_out, as bytes.  Fibres of len <= DAB_SORTPERM_SLICES_SMEM_LEN are sorted in shared memory by a bitonic
 * network over (radix key, position) pairs; longer fibres take two chunk-wide stable K21 passes (by key, then by fibre id) whatever the
 * number of fibres, with scratch from the ctx block cache, and need a chunk of fewer than 2^32 - 4096 elements (otherwise
 * DAB_ERR_UNSUPPORTED).  DAB_ERR_ARG: chunk_dims[dim-1] != global_dims[dim-1], a chunk outside the array, or a NULL pointer;
 * DAB_ERR_UNSUPPORTED: key dtypes other than F32 F64 I32 I64, ndim > 8.  keys and vals are only read; perm / vals_out must not overlap
 * them.  An empty chunk launches nothing.  Asynchronous on the ctx stream. */
#define DAB_SORTPERM_SLICES_SMEM_LEN 4096
int32_t dab_sortperm_slices(dab_ctx* ctx, int32_t key_dtype, const void* keys, int32_t ndim, const size_t* chunk_dims, const size_t* chunk_lo,
                            const size_t* global_dims, int32_t dim, int64_t* perm, int32_t val_bytes, const void* vals, void* vals_out);

/* Limits of dab_svdvals_batched: min(m, n) and m * n. */
#define DAB_SVDVALS_MAX_K 32
#define DAB_SVDVALS_MAX_ELEMS 4096
/* S[b*k .. b*k + k) = svdvals(A_b), descending, k = min(m, n), for the `batch` dense column-major m x n matrices A_b stored one after the
 * other: mapslices(svdvals, lp, dims=(d1, d2)) once the slices are packed.  One-sided Jacobi in fp64 (Float32 input is rounded once at
 * the end).  dtypes F32 F64; min(m, n) <= DAB_SVDVALS_MAX_K and m * n <= DAB_SVDVALS_MAX_ELEMS, otherwise DAB_ERR_UNSUPPORTED.  status: a
 * device int32 set to 0 by the call and to 1 by the kernel when a matrix holds a NaN or Inf (its values are then NaN); Julia's LAPACK
 * wrapper rejects such input (chkfinite), so the host runtime raises ArgumentError once it has read status. */
int32_t dab_svdvals_batched(dab_ctx* ctx, int32_t dtype, const void* A, size_t m, size_t n, size_t batch, void* S, int32_t* status);

/* The slice functions of ppeval(f, D...; dim) (src/mapreduce.jl:210-323) that need a kernel of their own: the  _ppeval(f, localparts...)
 * run on every worker (:315) once the slices are packed. */

/* C_b = A_b * B_b for b < batch: A_b is m x k at A + b * strideA, B_b is k x n at B + b * strideB, C_b is m x n at C + b * m * n, all dense
 * column-major; strides in elements, 0 broadcasts that operand to every b.  ppeval(*, A, B) with A_b, B_b the slices.  Float32 products
 * accumulate in fp64 and are rounded once; Float64 accumulates with one DFMA per k, in k order; Int32 / Int64 wrap as Julia's generic
 * matmul (Int32 results are Int32).  k == 0 writes zeros.  C must not overlap A or B.  dtypes F32 F64 I32 I64. */
int32_t dab_matmul_batched(dab_ctx* ctx, int32_t dtype, size_t m, size_t n, size_t k, const void* A, size_t strideA, const void* B,
                           size_t strideB, void* C, size_t batch);

/* Largest n dab_eigvals_sym_batched serves (one 32 KiB fp64 matrix in shared memory). */
#define DAB_EIGVALS_SYM_MAX_N 64
/* W[b*n .. b*n + n) = eigvals(A_b), ascending, for the `batch` dense column-major n x n matrices A_b stored one after the other:
 * ppeval(eigvals, D) / mapslices(eigvals, lp, dims=(d1, d2)) once the slices are packed.  Two-sided cyclic Jacobi in fp64 (Float32 input
 * is rounded once at the end).  dtypes F32 F64; n <= DAB_EIGVALS_SYM_MAX_N, otherwise DAB_ERR_UNSUPPORTED.  status: a device int32 set
 * to 0 by the call; the kernel ORs in 1 when a matrix holds a NaN or Inf and 2 when a finite matrix is not exactly symmetric
 * (A[i,j] != A[j,i]); that matrix's values are then NaN.  Julia rejects non-finite input (ArgumentError) and takes a non-symmetric
 * matrix to the general, complex eigenvalue problem, so the host runtime raises on either once it has read status. */
int32_t dab_eigvals_sym_batched(dab_ctx* ctx, int32_t dtype, const void* A, size_t n, size_t batch, void* W, int32_t* status);

/* Largest n dab_ldiv_batched / dab_det_batched serve (one fp64 matrix of a CTA's shared memory). */
#define DAB_LU_MAX_N 64
/* X_b = A_b \ B_b for b < batch: A_b n x n, B_b and X_b n x nrhs, dense column-major; strides in elements, 0 broadcasts that operand to
 * every b; X_b is stored at X + b*n*nrhs and must not overlap A or B, which are only read.  ppeval(\, A, B) once the slices are packed.
 * Julia's dispatch of `\` on a square matrix: a diagonal slice gives b ./ d (bit-exact), a lower or upper triangular one is solved by
 * substitution, any other is factored with partial pivoting (LAPACK's idamax rule) and solved with the factors.  fp64 throughout, Float32
 * rounded once.  status: a device uint64 set to all ones by the call; a failing slice b lowers it (atomicMin) to (b << 8) | low, with low =
 * info (1-based) for an exactly-zero diagonal entry or pivot (Julia's SingularException(info); not raised by a diagonal slice when nrhs == 0)
 * or 0x80 for a NaN / Inf anywhere in a slice on the LU path (ArgumentError from getrf!'s chkfinite; on the other paths NaN / Inf flow
 * through).  The word ends as the lowest failing b; X is unspecified for failing slices.  dtypes F32 F64 and n <= DAB_LU_MAX_N, otherwise
 * DAB_ERR_UNSUPPORTED before anything is launched.  n == 0 or batch == 0 launches nothing. */
int32_t dab_ldiv_batched(dab_ctx* ctx, int32_t dtype, size_t n, size_t nrhs, const void* A, size_t strideA, const void* B, size_t strideB,
                         void* X, size_t batch, void* status);
/* D[b] = det(A_b) for b < batch, A_b n x n dense column-major at A + b*strideA (0 broadcasts): ppeval(det, D) / mapslices(det, lp,
 * dims=(d1, d2)) once the slices are packed.  A triangular slice gives the product of its diagonal in index order; any other is factored
 * with partial pivoting and gives the product of U's diagonal in index order, negated for an odd number of row swaps, or +0.0 when a pivot
 * is exactly zero.  No finiteness check, no status: det never fails.  fp64 throughout, Float32 rounded once; n == 0 gives 1.  dtypes F32
 * F64 and n <= DAB_LU_MAX_N, otherwise DAB_ERR_UNSUPPORTED. */
int32_t dab_det_batched(dab_ctx* ctx, int32_t dtype, size_t n, const void* A, size_t strideA, void* D, size_t batch);

/* ==== cross-worker combine: NCCL over NVLink (replaces Distributed.remotecall_fetch on
 *      this path only; src/mapreduce.jl:30-34, 72-80; src/darray.jl:809-815) ============== */
/* 128-byte ncclUniqueId; rank 0 creates it, the host runtime ships it to the other workers. */
int32_t dab_comm_unique_id(void* id128);
int32_t dab_comm_init_rank(dab_ctx* ctx, const void* id128, int32_t rank, int32_t nranks);
int32_t dab_comm_destroy(dab_ctx* ctx);
/* asyncmap(procs(d)) do p; remotecall_fetch(...) end  -> every rank gets all P partials (device). */
int32_t dab_allgather(dab_ctx* ctx, const void* send_dev, void* recv_dev, size_t nbytes_per_rank);
int32_t dab_allreduce(dab_ctx* ctx, int32_t dtype, int32_t op, const void* send_dev, void* recv_dev, size_t count);
/* point-to-point slab / partial-vector transfer inside a group (mapreducedim_between!, halo). */
int32_t dab_group_start(dab_ctx* ctx);
int32_t dab_group_end(dab_ctx* ctx);
int32_t dab_send(dab_ctx* ctx, const void* send_dev, size_t nbytes, int32_t peer);
int32_t dab_recv(dab_ctx* ctx, void* recv_dev, size_t nbytes, int32_t peer);
/* sum(d) in one call: chunk reduce (dab_reduce) -> allgather of the P chunk results -> ordered left
 * fold (dab_combine_ordered) -> host scalar.  Exactly src/mapreduce.jl:29-35.  out_host: 8 bytes, 16 for a ComplexF64 result.
 * Complex results always take the dab_reduce + allgather + dab_combine_ordered path (the fused mailbox combine below carries
 * 8-byte results). */
int32_t dab_mapreduce_all(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* map_param, const void* x,
                          size_t n, void* out_host);

/* Fused reduce + combine over NVLink peer memory.  After every rank has created its mailbox (dab_mailbox_create returns the
 * 64-byte CUDA IPC handle), exchanged the handles through the host runtime and attached them (handles = nranks * 64 bytes, in
 * rank order), dab_mapreduce_all runs as ONE kernel: the last CTA of the chunk reduction pushes the chunk result into every
 * peer's mailbox with peer stores, waits for the P results, folds them left to right in rank order and writes the scalar into
 * pinned host memory -- no NCCL call, no D2H copy.  A rank that never calls makes the others time out (wall clock, default 120 s, dab_set_option "combine_timeout_ms") with DAB_ERR_NCCL
 * instead of hanging the GPU.  All ranks must call dab_mapreduce_all in the same order (as with any collective). */
int32_t dab_mailbox_create(dab_ctx* ctx, void* handle64);
int32_t dab_mailbox_attach(dab_ctx* ctx, const void* handles, int32_t rank, int32_t nranks);
int32_t dab_mailbox_detach(dab_ctx* ctx);

/* Device-side barrier across the ranks, ordered on the ctx stream (needs the mailboxes above; a no-op for one rank): kernels queued
 * after it start only when every rank's kernels queued before ITS call have completed.  The fence around one-sided peer reads / writes
 * (the remotecall_wait of the reference) without a host synchronisation or an NCCL launch; a peer that never arrives surfaces as
 * DAB_ERR_NCCL at the next dab_sync after "combine_timeout_ms". */
int32_t dab_peer_barrier(dab_ctx* ctx);
/* y = beta*y (fill!(0) when *beta == 0, untouched when 1), then y += alpha * stack[j*stride .. +n) for j = 0..count-1 in order, every
 * multiply and add rounded separately: rmul!/fill! + add!(localpart(y), R[i,j], alpha) of mul! (src/linalg.jl:101-117, 62-76; also the
 * between-phase of a sum over slabs) in one launch.  alpha, beta: host scalars of dtype (F32 F64 I32 I64). */
int32_t dab_accumulate_stack(dab_ctx* ctx, int32_t dtype, void* y, size_t n, const void* beta, const void* alpha, const void* stack,
                             size_t stride, int32_t count);

/* ==== peer memory (one process per GPU): CUDA IPC handles, shipped by the host runtime ==== */
int32_t dab_ipc_get_handle(dab_ctx* ctx, const void* dptr, void* handle64);
int32_t dab_ipc_open(dab_ctx* ctx, const void* handle64, void** dptr);
int32_t dab_ipc_close(dab_ctx* ctx, void* dptr);
/* in-process multi-GPU: enable peer access from ctx's device to `peer_device`. */
int32_t dab_enable_peer(dab_ctx* ctx, int32_t peer_device);

#ifdef __cplusplus
}
#endif
#endif /* DAB200_H */
