// dab_sort.cu -- K11: sort of one chunk, the `sort(localpart(d))` / `sort!(lp_sorting)` steps of the reference's samplesort
// (src/sort.jl:3-15, 18-63), and the split-point search of scatter_n_sort_localparts (:28-40).
//
// Keys only, ascending in Julia's `isless` order: integers by value; floats with -0.0 < +0.0 and every NaN after +Inf (bit
// patterns preserved; the reference keeps NaNs in their original relative order, here they are ordered by payload).
//
// Algorithm: least-significant-digit radix sort, 8-bit digits, hand-written for sm_90a, "onesweep" structure.  HBM-bound integer work:
//   sort_hist_kernel      one read of the keys -> the 256-bin histogram of EVERY digit position
//   sort_plan_kernel      (1 CTA) bucket bases per digit, which passes run (a digit that is constant over the chunk is skipped: Int64 data
//                         in a small range needs 2-3 of 8 passes), buffer ping-pong -- on the DEVICE: dab_sort never synchronises the stream
//   sort_onesweep_kernel  per remaining pass: ONE sweep = read the keys once, rank them inside the tile (ballots + per-warp shared counters,
//                         stable), resolve the tile's bucket offsets by decoupled look-back over the earlier tiles, reorder the tile by digit
//                         in shared memory and write it out in runs
// Algorithmic bytes: elem * (1 + 2 * passes) per key.
//
// K21, the pair sort (dab_sort_pairs, the kernel under sortperm): the same kernels with the payload parameter P = uint32_t.  Every key
// carries its 32-bit position in the chunk through the passes: the reorder step writes it to the same shared-memory slot as its key and
// the write-out moves both.  The first pass reads no payload (it generates the tile position), the last one writes the Int64 value
// (base + position, or vals[position]).  The radix key is sortby_radix_key: every NaN collapses to the top key, so NaNs are ties and
// LSD stability keeps them, like every other run of equal keys, in input order.  P = void is the keys-only K11, unchanged.
#include <map>
#include <mutex>
#include <type_traits>
#include <utility>

#include "dab_common.cuh"
#include "dab_sort_key.cuh"
#include "dab_sortby_core.cuh"

namespace {

// What the pair instances need beyond the keys; empty for the keys-only ones.
template <typename P> struct PairIO {};
template <> struct PairIO<uint32_t> {
    uint32_t* pos_out;       // positions between passes, beside the keys in `out`
    uint32_t* pos_tmp;       // ... beside the keys in `tmp`
    const int64_t* vals;     // NULL: the value of position i is base + i
    int64_t base;
    int64_t* vals_out;
    __device__ __forceinline__ int64_t value(uint32_t pos) const { return vals ? vals[pos] : base + (int64_t)pos; }
};

// Radix key of a raw key: the keys-only bijection, or (pairs) the same with every NaN collapsed to the top key.
template <typename T, typename P>
__device__ __forceinline__ typename SortKey<T>::U radix_of(typename SortKey<T>::U raw) {
    if constexpr (std::is_void<P>::value) return SortKey<T>::enc(raw);
    else return sortby_radix_key<T>(raw);
}

constexpr int ST_THREADS = 256;
constexpr int ST_KPT = 8;                        // keys per thread (16 left the scatter at 111 registers = 2 CTAs per SM, latency-bound)
constexpr int ST_TILE = ST_THREADS * ST_KPT;     // 2048 keys per CTA

// Lanes of the warp whose 8-bit digit equals mine (dg = 256 marks "no key"; those lanes group together): 9 ballots.  On sm_90a
// __match_any_sync costs one round per DISTINCT value in the warp (measured ~45 clk per warp-step on random digits); the bitwise
// form is flat.
template <int B>
__device__ __forceinline__ unsigned int match_bit(unsigned int dg, unsigned int m) {
    // 4 instructions per bit (LOP3 -> predicate, VOTE, SEL, LOP3); the C++ spelling compiles to 6
    unsigned int bal, inv;
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .u32 t;\n\t"
        "and.b32 t, %2, %3;\n\t"
        "setp.ne.u32 p, t, 0;\n\t"
        "vote.sync.ballot.b32 %0, p, 0xffffffff;\n\t"
        "selp.u32 %1, 0, 0xffffffff, p;\n\t}"
        : "=r"(bal), "=r"(inv)
        : "r"(dg), "n"(1u << B));
    return m & (bal ^ inv);
}
template <int BITS>
__device__ __forceinline__ unsigned int match_digit(unsigned int dg) {
    unsigned int m = 0xffffffffu;
    m = match_bit<0>(dg, m);
    m = match_bit<1>(dg, m);
    m = match_bit<2>(dg, m);
    m = match_bit<3>(dg, m);
    m = match_bit<4>(dg, m);
    m = match_bit<5>(dg, m);
    m = match_bit<6>(dg, m);
    m = match_bit<7>(dg, m);
    if (BITS > 8) m = match_bit<8>(dg, m);
    return m;
}

// A thread's ST_KPT CONSECUTIVE keys (blocked arrangement: 128 contiguous bytes of 8-byte keys), 16-byte loads when the tile is full
// and aligned.  Returns how many of them exist.  Used by the counting kernels: runs of equal digits (sorted or narrow-range input)
// collapse into one shared-memory atomic per run instead of serialising a whole warp on one bin.
template <typename U>
__device__ __forceinline__ int load_blocked(const U* __restrict__ in, size_t first, size_t n, U (&key)[ST_KPT]) {
    if (first + ST_KPT <= n && (reinterpret_cast<uintptr_t>(in) & 15u) == 0) {
        constexpr int PER = 16 / sizeof(U);
        const int4* p = reinterpret_cast<const int4*>(in + first);
#pragma unroll
        for (int q = 0; q < ST_KPT / PER; ++q) {
            const int4 v = __ldcs(p + q);
            memcpy(&key[q * PER], &v, 16);
        }
        return ST_KPT;
    }
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < ST_KPT; ++k)
        if (first + k < n) {
            key[k] = __ldcs(in + first + k);
            cnt = k + 1;
        }
    return cnt;
}

// ---- all-digit histogram ------------------------------------------------------------------------------------------------------------
template <typename T, typename P>
__global__ void __launch_bounds__(ST_THREADS) sort_hist_kernel(const typename SortKey<T>::U* __restrict__ in, size_t n,
                                                               unsigned long long* __restrict__ ghist) {
    using K = SortKey<T>;
    using U = typename K::U;
    __shared__ unsigned int sh[K::DIGITS][256];
    for (int i = threadIdx.x; i < K::DIGITS * 256; i += ST_THREADS) (&sh[0][0])[i] = 0;
    __syncthreads();
    // grid-stride over tiles: a few CTAs per SM accumulate privately, so the global histogram sees gridDim.x flushes, not n / 4096
    for (size_t base = (size_t)blockIdx.x * ST_TILE; base < n; base += (size_t)gridDim.x * ST_TILE) {
        U key[ST_KPT];
        const int cnt = load_blocked<U>(in, base + (size_t)threadIdx.x * ST_KPT, n, key);
        if (cnt > 0) {
            unsigned int cur[K::DIGITS], run[K::DIGITS];
            const U k0 = radix_of<T, P>(key[0]);
#pragma unroll
            for (int d = 0; d < K::DIGITS; ++d) {
                cur[d] = (unsigned)(k0 >> (8 * d)) & 255u;
                run[d] = 1;
            }
#pragma unroll
            for (int k = 1; k < ST_KPT; ++k)
                if (k < cnt) {
                    const U kk = radix_of<T, P>(key[k]);
#pragma unroll
                    for (int d = 0; d < K::DIGITS; ++d) {
                        const unsigned int dg = (unsigned)(kk >> (8 * d)) & 255u;
                        if (dg == cur[d]) {
                            ++run[d];
                        } else {
                            atomicAdd(&sh[d][cur[d]], run[d]);
                            cur[d] = dg;
                            run[d] = 1;
                        }
                    }
                }
#pragma unroll
            for (int d = 0; d < K::DIGITS; ++d) atomicAdd(&sh[d][cur[d]], run[d]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K::DIGITS * 256; i += ST_THREADS) {
        const unsigned int c = (&sh[0][0])[i];
        if (c) atomicAdd(ghist + i, (unsigned long long)c);
    }
}

// ---- the device-side plan: which digit passes run, and from/to which buffer -----------------------------------------------------------
// Everything the round-1 host code decided after reading the histograms back is decided here on the device, so dab_sort never
// synchronises the stream: constant digits are skipped (Int64 keys in 0:10^6 need 3 of 8 passes), the buffers ping-pong so that the
// LAST active pass writes `out`, an in-place sort with an odd number of passes stages its input in `tmp` first.
enum { SEL_IN = 0, SEL_OUT = 1, SEL_TMP = 2 };
struct SortPlan {
    unsigned long long hist[8][256];   // all-digit histograms (sort_hist_kernel)
    unsigned int base[8][256];         // exclusive scan of each histogram: first output slot of every bucket
    unsigned int tile_ticket[8];       // per pass: the next tile to hand out (tiles are taken in address order)
    int active[8], src_sel[8], dst_sel[8];
    int raw_in[8], raw_out[8];         // first active pass reads raw keys, last one writes raw keys; in between the keys stay encoded
    int n_active, precopy;             // precopy: in-place sort, odd pass count -> copy in to tmp before the first pass
};

template <int DIGITS>
__global__ void __launch_bounds__(256) sort_plan_kernel(SortPlan* plan, unsigned long long n, int inplace) {
    __shared__ unsigned long long wsum[8];
    __shared__ int constant[8];
    const int b = threadIdx.x, lane = b & 31, warp = b >> 5;
    if (b < 8) constant[b] = 0;
    __syncthreads();
    for (int d = 0; d < DIGITS; ++d) {
        const unsigned long long h = plan->hist[d][b];
        if (h == n) constant[d] = 1;
        unsigned long long inc = h;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, s);
            if (lane >= s) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        unsigned long long carry = 0;
        for (int w = 0; w < warp; ++w) carry += wsum[w];
        plan->base[d][b] = (unsigned int)(carry + inc - h);
        __syncthreads();
    }
    if (b == 0) {
        int na = 0;
        for (int d = 0; d < DIGITS; ++d) na += !constant[d];
        int q = 0, prev = SEL_IN, pre = 0;
        for (int d = 0; d < 8; ++d) {
            plan->tile_ticket[d] = 0;
            const int act = d < DIGITS && !constant[d];
            plan->active[d] = act;
            if (!act) continue;
            const int dst = ((na - 1 - q) % 2 == 0) ? SEL_OUT : SEL_TMP;
            int src = prev;
            if (q == 0 && inplace && dst == SEL_OUT) {   // in == out and the first pass would overwrite its own input
                pre = 1;
                src = SEL_TMP;
            }
            plan->src_sel[d] = src;
            plan->dst_sel[d] = dst;
            plan->raw_in[d] = q == 0;
            plan->raw_out[d] = q == na - 1;
            prev = dst;
            ++q;
        }
        plan->n_active = na;
        plan->precopy = pre;
    }
}

// mode 0: copy in -> tmp when the plan asks for the staging copy; mode 1: copy in -> out when NO pass runs (all keys equal; pairs: the
// permutation is the identity, so vals_out gets the values in input order, and an in-place sort copies no key)
template <typename U, typename P>
__global__ void __launch_bounds__(256) sort_copy_if_kernel(const SortPlan* __restrict__ plan, const U* __restrict__ src, U* __restrict__ dst,
                                                           size_t n, int mode, PairIO<P> io) {
    if (mode == 0 ? !plan->precopy : plan->n_active != 0) return;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
        if constexpr (std::is_void<P>::value) {
            dst[i] = src[i];
        } else {
            if (src != dst) dst[i] = src[i];
            if (mode == 1) io.vals_out[i] = io.value((uint32_t)i);
        }
    }
}

// ---- one digit pass, "onesweep": count + look-back + stable scatter in ONE sweep over the keys ------------------------------------------
// Per pass each key is read once and written once (round 1: read twice, written once, plus a scan launch).  A persistent CTA takes tiles
// by ticket (address order, so the look-back below always waits on a tile that is already running):
//   1. all KPT loads of a thread are issued before any use (full tiles: unpredicated, so ptxas does not sink them into the ranking loop)
//   2. ranking: warp w owns a contiguous run; equal digits inside a 32-key step are grouped by ballots, a per-warp shared counter row
//      carries the running rank -> stable
//   3. thread d publishes the tile's count of digit d (PARTIAL), then walks back over the predecessors' words until it meets an INCLUSIVE
//      one: decoupled look-back, one 64-bit word = flag | epoch | count, so no fence is needed and the scratch is never cleared (a word of
//      an older pass carries an older epoch and reads as "not ready")
//   4. the tile is reordered by digit in shared memory, then written out: consecutive threads -> consecutive addresses inside each
//      bucket run (full 32-byte sectors instead of one sector request per key)
constexpr unsigned long long LB_PARTIAL = 1ull << 62, LB_INCLUSIVE = 2ull << 62, LB_FLAGS = 3ull << 62;
constexpr unsigned long long LB_EPOCH_MASK = ((1ull << 30) - 1ull) << 32;
constexpr int LB_WINDOW = 8;   // predecessor words fetched per look-back round (independent L2 reads in flight instead of a serial walk)

__device__ __forceinline__ uint32_t sort_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Ranks of a warp's KPT x 32 keys among the keys of the same digit seen so far by this warp (stable).  Equal digits inside a 32-key step
// are grouped by ballots; the group's lowest lane bumps the warp's shared counter of that digit once (predicated ATOMS, no divergent branch)
// and hands the old value round; the steps are issued in order by the one warp that owns the counter row.
template <typename T, int KPT, bool FULL>
__device__ __forceinline__ void onesweep_rank(const typename SortKey<T>::U* __restrict__ stage, unsigned int wofs, int lane, unsigned int lt,
                                              unsigned int nvalid, int shift, uint32_t wc_row, unsigned short (&rank)[KPT]) {
    using U = typename SortKey<T>::U;
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const unsigned int li = wofs + (unsigned)k * 32 + lane;
        const bool valid = FULL || li < nvalid;
        const U key = stage[li];
        const unsigned int dg = valid ? ((unsigned)(key >> shift) & 255u) : 256u;   // missing keys form their own group
        const unsigned int grp = match_digit<FULL ? 8 : 9>(dg);
        const unsigned int before = __popc(grp & lt);
        const int leader = __ffs(grp) - 1;
        unsigned int old = 0;
        const unsigned int gsize = __popc(grp);
        const unsigned int doit = (valid && before == 0) ? 1u : 0u;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.u32 p, %3, 0;\n\t"
            "@p atom.shared.add.u32 %0, [%1], %2;\n\t}"
            : "+r"(old)
            : "r"(wc_row + dg * 4u), "r"(gsize), "r"(doit));
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[k] = (unsigned short)(old + before);
    }
}

// The tile, sorted by the digit, into the second shared-memory buffer: local slot = start of the digit's run for this warp + rank.
// Pairs: the key's position goes to the same slot of the position buffer -- pstage[li], or tbase + li when the pass generates it.
template <typename T, typename P, int KPT, bool FULL>
__device__ __forceinline__ void onesweep_reorder(const typename SortKey<T>::U* __restrict__ stage, uint32_t sorted_s, unsigned int wofs, int lane,
                                                 unsigned int nvalid, int shift, uint32_t wc_row, const unsigned short (&rank)[KPT],
                                                 const uint32_t* __restrict__ pstage, uint32_t psorted_s, bool gen_pos, unsigned int tbase) {
    using U = typename SortKey<T>::U;
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const unsigned int li = wofs + (unsigned)k * 32 + lane;
        if (FULL || li < nvalid) {
            const U key = stage[li];
            const unsigned int dg = (unsigned)(key >> shift) & 255u;
            unsigned int base;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(base) : "r"(wc_row + dg * 4u));
            const uint32_t a = sorted_s + (base + rank[k]) * (unsigned)sizeof(U);
            if constexpr (sizeof(U) == 8) asm volatile("st.shared.b64 [%0], %1;" ::"r"(a), "l"(key) : "memory");
            else asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(key) : "memory");
            if constexpr (!std::is_void<P>::value) {
                const uint32_t pos = gen_pos ? tbase + li : pstage[li];
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(psorted_s + (base + rank[k]) * 4u), "r"(pos) : "memory");
            }
        }
    }
}

// One digit pass over the whole chunk.  Persistent CTAs take tiles by ticket; per tile:
//   stage   the tile's keys arrive in shared memory by ONE bulk async copy (cp.async.bulk, the TMA engine; SASS UBLKCP) issued by one
//           thread and completing on an mbarrier -- issued for the NEXT tile as soon as the current one has been reordered, so the DRAM
//           latency of tile t+1 hides behind the look-back and the write-out of tile t (plain loads only for a misaligned or ragged tile)
//   rank    warp w owns a contiguous run; equal digits inside a 32-key step are grouped by ballots, a per-warp shared counter row carries
//           the running rank (stable).  Keys are re-read from shared memory, so a thread holds 16-bit ranks, not keys, in registers.
//   publish thread d sends the tile's count of digit d (PARTIAL) at once; decoupled look-back resolves the exclusive prefix later
//   reorder the tile is written, sorted by digit, into a second shared-memory buffer
//   write   consecutive threads -> consecutive addresses inside each bucket run
// Pairs (P = uint32_t): the positions travel in two more shared buffers beside the keys, by a second bulk copy on the same mbarrier.
template <typename T, typename P, int THREADS, int KPT, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) sort_onesweep_kernel(const typename SortKey<T>::U* __restrict__ in, typename SortKey<T>::U* __restrict__ out,
                                                                      typename SortKey<T>::U* __restrict__ tmp, size_t n, int d, SortPlan* __restrict__ plan,
                                                                      unsigned long long* __restrict__ lookback, unsigned int ntiles,
                                                                      unsigned long long epoch, PairIO<P> io) {
    using K = SortKey<T>;
    using U = typename K::U;
    constexpr bool PAIRS = !std::is_void<P>::value;
    constexpr int WARPS = THREADS / 32;
    constexpr int TILE = THREADS * KPT;
    static_assert(THREADS >= 256 && THREADS % 32 == 0, "thread d serves digit d");
    if (!plan->active[d]) return;
    extern __shared__ __align__(128) unsigned char os_smem[];
    U* stage = reinterpret_cast<U*>(os_smem);                                   // [TILE] the tile as it sits in memory
    U* sorted = stage + TILE;                                                   // [TILE] the tile sorted by the digit
    uint32_t* pstage = reinterpret_cast<uint32_t*>(sorted + TILE);              // pairs: [TILE] positions of `stage`
    uint32_t* psorted = pstage + TILE;                                          // pairs: [TILE] positions of `sorted`
    unsigned int (*wc)[256] = reinterpret_cast<unsigned int (*)[256]>(PAIRS ? psorted + TILE : pstage);   // [WARPS][256]
    unsigned int* dbase = &wc[WARPS][0];                                        // [256]
    unsigned int* wtot = dbase + 256;                                           // [8]
    __shared__ unsigned int s_next;
    __shared__ __align__(8) unsigned long long s_bar;
    const int ssel = plan->src_sel[d], dsel = plan->dst_sel[d];
    const U* __restrict__ src = ssel == SEL_IN ? in : (ssel == SEL_OUT ? out : tmp);
    U* __restrict__ dst = dsel == SEL_OUT ? out : tmp;
    const bool raw_in = plan->raw_in[d] != 0, raw_out = plan->raw_out[d] != 0;   // buffers between passes hold ENCODED keys
    // pairs: positions come from the buffer beside the source keys (none on the first pass: it generates them) and go beside the
    // destination keys (the last pass writes the Int64 values instead)
    const uint32_t* __restrict__ psrc = nullptr;
    uint32_t* __restrict__ pdst = nullptr;
    if constexpr (PAIRS) {
        psrc = raw_in ? nullptr : (ssel == SEL_OUT ? io.pos_out : io.pos_tmp);
        pdst = dsel == SEL_OUT ? io.pos_out : io.pos_tmp;
    }
    const unsigned int* gbase = plan->base[d];
    const int shift = 8 * d;
    const unsigned long long ep = (epoch << 32) & LB_EPOCH_MASK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int lt = (1u << lane) - 1u;
    const bool src_aligned = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
    const uint32_t bar = sort_smem_u32(&s_bar), stage_s = sort_smem_u32(stage), sorted_s = sort_smem_u32(sorted);
    const uint32_t wc_row = sort_smem_u32(&wc[warp][0]);
    const uint32_t pstage_s = sort_smem_u32(pstage), psorted_s = sort_smem_u32(psorted);
    // a tile can come by bulk copy when its bytes are a multiple of 16 from a 16-byte aligned address (pairs: its positions too)
    auto bulk_ok = [&](unsigned int t) -> bool {
        if (!src_aligned) return false;
        const size_t tb = (size_t)t * TILE;
        const size_t cnt = (tb + TILE <= n) ? (size_t)TILE : n - tb;
        if constexpr (PAIRS)
            if (psrc && (cnt % 4 != 0 || (reinterpret_cast<uintptr_t>(psrc) & 15u) != 0)) return false;
        return (cnt * sizeof(U)) % 16 == 0;
    };
    auto issue_bulk = [&](unsigned int t) {   // one thread
        const size_t tb = (size_t)t * TILE;
        const uint32_t bytes = (uint32_t)(((tb + TILE <= n) ? (size_t)TILE : n - tb) * sizeof(U));
        if constexpr (PAIRS) {
            const uint32_t pbytes = psrc ? bytes / (uint32_t)sizeof(U) * 4u : 0u;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes + pbytes) : "memory");
            if (pbytes)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(pstage_s), "l"(psrc + tb), "r"(pbytes), "r"(bar)
                             : "memory");
        } else {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        }
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(stage_s), "l"(src + tb), "r"(bytes), "r"(bar)
                     : "memory");
    };
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned int t0 = atomicAdd(&plan->tile_ticket[d], 1u);
        s_next = t0;
        if (t0 < ntiles && bulk_ok(t0)) issue_bulk(t0);
    }
    unsigned int phase = 0;
    for (;;) {
        for (int i = threadIdx.x; i < WARPS * 256; i += THREADS) (&wc[0][0])[i] = 0;
        __syncthreads();                                        // s_next, zeroed counters, mbarrier init
        const unsigned int tile = s_next;
        if (tile >= ntiles) return;
        const size_t tbase = (size_t)tile * TILE;
        const bool full = tbase + TILE <= n;
        const unsigned int nvalid = full ? (unsigned)TILE : (unsigned)(n - tbase);
        if (bulk_ok(tile)) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "W_%=:\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                "@!p bra W_%=;\n\t}"
                ::"r"(bar), "r"(phase)
                : "memory");
            phase ^= 1u;
        } else {                                                // misaligned source or ragged byte count: plain loads by everybody
            for (unsigned int i = threadIdx.x; i < nvalid; i += THREADS) stage[i] = __ldcs(src + tbase + i);
            if constexpr (PAIRS)
                if (psrc)
                    for (unsigned int i = threadIdx.x; i < nvalid; i += THREADS) pstage[i] = __ldcs(psrc + tbase + i);
            __syncthreads();
        }
        const unsigned int wofs = (unsigned)warp * (KPT * 32);
        if (raw_in) {   // first pass only: encode the thread's own keys in place, so that ranking and reordering read encoded keys
#pragma unroll
            for (int k = 0; k < KPT; ++k) {
                const unsigned int li = wofs + (unsigned)k * 32 + lane;
                if (full || li < nvalid) stage[li] = radix_of<T, P>(stage[li]);
            }
        }
        unsigned short rank[KPT];
        if (full) onesweep_rank<T, KPT, true>(stage, wofs, lane, lt, nvalid, shift, wc_row, rank);
        else onesweep_rank<T, KPT, false>(stage, wofs, lane, lt, nvalid, shift, wc_row, rank);
        __syncthreads();
        unsigned int cnt = 0, tstart = 0;
        unsigned long long* myword = nullptr;
        if (threadIdx.x < 256) {
            const int dd = threadIdx.x;
            // running prefix of digit dd over the warps; the tile's count goes out at once so that successors can make progress
#pragma unroll
            for (int w = 0; w < WARPS; ++w) {
                const unsigned int c = wc[w][dd];
                wc[w][dd] = cnt;
                cnt += c;
            }
            myword = lookback + (size_t)tile * 256 + dd;
            *(volatile unsigned long long*)myword = (tile == 0 ? LB_INCLUSIVE : LB_PARTIAL) | ep | (unsigned long long)cnt;
            // exclusive scan of the 256 digit counts -> where digit dd starts inside the sorted tile
            unsigned int inc = cnt;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, inc, s);
                if (lane >= s) inc += t;
            }
            if (lane == 31) wtot[warp] = inc;
            tstart = inc - cnt;
        }
        __syncthreads();
        if (threadIdx.x < 256) {
            for (int w = 0; w < warp; ++w) tstart += wtot[w];
            const int dd = threadIdx.x;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) wc[w][dd] += tstart;
        }
        __syncthreads();
        if (full) onesweep_reorder<T, P, KPT, true>(stage, sorted_s, wofs, lane, nvalid, shift, wc_row, rank, pstage, psorted_s, raw_in, (unsigned)tbase);
        else onesweep_reorder<T, P, KPT, false>(stage, sorted_s, wofs, lane, nvalid, shift, wc_row, rank, pstage, psorted_s, raw_in, (unsigned)tbase);
        __syncthreads();                                        // `stage` is free again, `sorted` is complete
        if (threadIdx.x == 0) {                                 // next tile: ticket + bulk copy, in flight during look-back and write-out
            const unsigned int t1 = atomicAdd(&plan->tile_ticket[d], 1u);
            s_next = t1;
            if (t1 < ntiles && bulk_ok(t1)) issue_bulk(t1);
        }
        if (threadIdx.x < 256) {
            const int dd = threadIdx.x;
            unsigned int excl = 0;
            if (tile > 0) {
                long long t = (long long)tile - 1;   // next predecessor to consume
                bool done = false;
                while (!done) {
                    unsigned long long v[LB_WINDOW];
#pragma unroll
                    for (int j = 0; j < LB_WINDOW; ++j)
                        v[j] = (t - j >= 0) ? *(const volatile unsigned long long*)(lookback + (size_t)(t - j) * 256 + dd) : (LB_INCLUSIVE | ep);
#pragma unroll
                    for (int j = 0; j < LB_WINDOW; ++j) {
                        if (done) break;
                        if ((v[j] & LB_FLAGS) == 0 || (v[j] & LB_EPOCH_MASK) != ep) break;   // not published yet: fetch again from here
                        excl += (unsigned int)v[j];
                        --t;
                        if (v[j] & LB_INCLUSIVE) done = true;
                    }
                }
                *(volatile unsigned long long*)myword = LB_INCLUSIVE | ep | (unsigned long long)(excl + cnt);
            }
            dbase[dd] = gbase[dd] + excl - tstart;
        }
        __syncthreads();
        if constexpr (PAIRS) {   // key and position leave together; the last pass turns the position into its Int64 value
            auto put = [&](unsigned int i) {
                const U kk = sorted[i];
                const unsigned int o = dbase[(unsigned)(kk >> shift) & 255u] + i;
                const uint32_t pos = psorted[i];
                if (raw_out) {
                    dst[o] = K::dec(kk);
                    io.vals_out[o] = io.value(pos);
                } else {
                    dst[o] = kk;
                    pdst[o] = pos;
                }
            };
            if (full) {
#pragma unroll
                for (int k = 0; k < KPT; ++k) put((unsigned)k * THREADS + threadIdx.x);
            } else {
                for (unsigned int i = threadIdx.x; i < nvalid; i += THREADS) put(i);
            }
        } else if (full && !raw_out) {
#pragma unroll
            for (int k = 0; k < KPT; ++k) {
                const unsigned int i = (unsigned)k * THREADS + threadIdx.x;
                const U kk = sorted[i];
                dst[dbase[(unsigned)(kk >> shift) & 255u] + i] = kk;
            }
        } else if (full) {   // last pass: back to the raw bit patterns
#pragma unroll
            for (int k = 0; k < KPT; ++k) {
                const unsigned int i = (unsigned)k * THREADS + threadIdx.x;
                const U kk = sorted[i];
                dst[dbase[(unsigned)(kk >> shift) & 255u] + i] = K::dec(kk);
            }
        } else {
            for (unsigned int i = threadIdx.x; i < nvalid; i += THREADS) {
                const U kk = sorted[i];
                dst[dbase[(unsigned)(kk >> shift) & 255u] + i] = raw_out ? K::dec(kk) : kk;
            }
        }
        // the loop top zeroes wc and syncs before anybody reads s_next / writes `sorted` again
    }
}

// encode / decode a whole buffer (only when no digit pass runs at all, or as the odd-parity fix-up never needed: kept for n small)
template <typename T, typename P>
__global__ void sort_small_kernel(const typename SortKey<T>::U* __restrict__ in, typename SortKey<T>::U* __restrict__ out, unsigned int n,
                                  PairIO<P> io) {
    // n <= 1024: rank sort in shared memory by one CTA (stable: ties broken by index)
    using K = SortKey<T>;
    using U = typename K::U;
    __shared__ U sk[1024];
    for (unsigned int i = threadIdx.x; i < n; i += blockDim.x) sk[i] = radix_of<T, P>(in[i]);
    __syncthreads();
    for (unsigned int i = threadIdx.x; i < n; i += blockDim.x) {
        const U me = sk[i];
        unsigned int r = 0;
        for (unsigned int j = 0; j < n; ++j) {
            const U o = sk[j];
            r += (o < me) || (o == me && j < i);
        }
        out[r] = K::dec(me);
        if constexpr (!std::is_void<P>::value) io.vals_out[r] = io.value(i);
    }
}

int32_t sort_scratch(dab_ctx* ctx, size_t dev_bytes) {
    if (!ctx->sort_host) DAB_CUDA(ctx, cudaMallocHost(&ctx->sort_host, 8 * 256 * sizeof(unsigned long long) + 4096));
    // the look-back words carry an epoch, so the scratch is cleared ONCE, when it is allocated (epoch 0 is never used by a pass)
    return dab_scratch_grow(ctx, &ctx->sort_dev, &ctx->sort_dev_bytes, dev_bytes, true);
}

constexpr size_t SORT_PLAN_BYTES = 65536;   // SortPlan + the staging areas of dab_sorted_split, ahead of the look-back words
static_assert(sizeof(SortPlan) + 8192 <= SORT_PLAN_BYTES, "plan area");

template <typename T, typename P, int THREADS, int KPT, int MINB>
int32_t sort_passes(dab_ctx* ctx, const typename SortKey<T>::U* in, typename SortKey<T>::U* out, typename SortKey<T>::U* tmp, size_t n,
                    PairIO<P> io) {
    using K = SortKey<T>;
    using U = typename K::U;
    constexpr bool PAIRS = !std::is_void<P>::value;
    constexpr int TILE = THREADS * KPT;
    const unsigned int ntiles = (unsigned int)((n + TILE - 1) / TILE);
    {
        int32_t st = sort_scratch(ctx, SORT_PLAN_BYTES + (size_t)ntiles * 256 * sizeof(unsigned long long));
        if (st != DAB_OK) return st;
    }
    SortPlan* plan = (SortPlan*)ctx->sort_dev;
    unsigned long long* lookback = (unsigned long long*)((char*)ctx->sort_dev + SORT_PLAN_BYTES);
    DAB_CUDA(ctx, cudaMemsetAsync(plan->hist, 0, sizeof(plan->hist), ctx->stream));
    {
        const unsigned int htiles = (unsigned int)((n + ST_TILE - 1) / ST_TILE);
        const unsigned int hgrid = htiles < (unsigned)ctx->sm_count * 4u ? htiles : (unsigned)ctx->sm_count * 4u;
        sort_hist_kernel<T, P><<<hgrid, ST_THREADS, 0, ctx->stream>>>(in, n, &plan->hist[0][0]);
        DAB_LAUNCHED(ctx);
    }
    const int inplace = (const void*)in == (const void*)out;
    sort_plan_kernel<K::DIGITS><<<1, 256, 0, ctx->stream>>>(plan, (unsigned long long)n, inplace);
    DAB_LAUNCHED(ctx);
    const int cgrid = dab_grid_for(ctx, (n + 1023) / 1024, 8);
    if (inplace) {
        sort_copy_if_kernel<U, P><<<cgrid, 256, 0, ctx->stream>>>(plan, in, tmp, n, 0, io);
        DAB_LAUNCHED(ctx);
    }
    if (!inplace || PAIRS) {   // acts only when every key is equal (pairs: vals_out is written even when the keys stay in place)
        sort_copy_if_kernel<U, P><<<cgrid, 256, 0, ctx->stream>>>(plan, in, out, n, 1, io);
        DAB_LAUNCHED(ctx);
    }
    auto kern = sort_onesweep_kernel<T, P, THREADS, KPT, MINB>;
    constexpr size_t smem = 2 * (size_t)TILE * (sizeof(U) + (PAIRS ? 4 : 0)) + (size_t)(THREADS / 32) * 1024 + 1024 + 32;
    int per_sm = 0;
    {   // >48 KiB of dynamic shared memory is an opt-in attribute of the (kernel, device) pair; the occupancy query needs it set
        static std::mutex mu;
        static std::map<std::pair<const void*, int>, int> seen;
        std::lock_guard<std::mutex> lk(mu);
        auto key = std::make_pair((const void*)kern, ctx->device);
        auto it = seen.find(key);
        if (it == seen.end()) {
            DAB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int nb = 0;
            DAB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, THREADS, smem));
            it = seen.emplace(key, nb < 1 ? 1 : nb).first;
        }
        per_sm = it->second;
    }
    const int grid = dab_grid_for(ctx, ntiles, per_sm);
    for (int d = 0; d < K::DIGITS; ++d) {
        const unsigned long long epoch = (++ctx->sort_epoch) & ((1ull << 30) - 1ull);
        if (epoch == 0) {   // wrapped (2^30 passes): start a new era with clean words
            DAB_CUDA(ctx, cudaMemsetAsync(lookback, 0, ctx->sort_dev_bytes - SORT_PLAN_BYTES, ctx->stream));
            --d;
            continue;
        }
        kern<<<grid, THREADS, smem, ctx->stream>>>(in, out, tmp, n, d, plan, lookback, ntiles, epoch, io);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

template <typename T, typename P = void>
int32_t sort_t(dab_ctx* ctx, const void* in_v, void* out_v, void* tmp_v, size_t n, PairIO<P> io = {}) {
    using K = SortKey<T>;
    using U = typename K::U;
    const U* in = (const U*)in_v;
    U* out = (U*)out_v;
    U* tmp = (U*)tmp_v;
    if (n == 0) return DAB_OK;
    if (n <= 1024) {
        const U* src = in;
        if (in == out) {  // the rank sort is not in-place
            DAB_REQUIRE(ctx, tmp != nullptr, DAB_ERR_ARG, "dab_sort: in-place sort needs tmp");
            DAB_CUDA(ctx, cudaMemcpyAsync(tmp, in, n * sizeof(U), cudaMemcpyDeviceToDevice, ctx->stream));
            src = tmp;
        }
        sort_small_kernel<T, P><<<1, 256, 0, ctx->stream>>>(src, out, (unsigned)n, io);
        DAB_LAUNCHED(ctx);
        return DAB_OK;
    }
    DAB_REQUIRE(ctx, tmp != nullptr && tmp != out && tmp != in, DAB_ERR_ARG, "dab_sort: tmp must be a distinct buffer of n elements");
    DAB_REQUIRE(ctx, n < 0xFFFFF000ull, DAB_ERR_UNSUPPORTED, "dab_sort: chunks of 2^32 or more elements are not served");
    // tile shape: 32 KiB of keys per CTA in shared memory -> ~128-byte bucket runs per tile on random digits
    // tile shape (tools/sort_vs_cub.cu sweeps it: larger tiles and 3 resident CTAs per SM won over smaller tiles at 4 CTAs
    // and over 128-register CTAs at 2): 256 threads x 16 keys (64-bit) / x 32 keys (32-bit) = 32 KiB of keys per tile, twice in shared memory
    // Pairs hold a 4-byte position beside every key, twice: the tiles shrink so that 3 CTAs per SM still fit (4096 pairs of 32-bit
    // keys = 64 KiB, 2560 pairs of 64-bit keys = 60 KiB, plus 9 KiB of counters each; 72 registers, no spills, -Xptxas -v)
    if constexpr (!std::is_void<P>::value) {
        if constexpr (sizeof(U) == 8) return sort_passes<T, P, 256, 10, 3>(ctx, in, out, tmp, n, io);
        else return sort_passes<T, P, 256, 16, 3>(ctx, in, out, tmp, n, io);
    } else if constexpr (sizeof(U) == 8) {
        return sort_passes<T, P, 256, 16, 3>(ctx, in, out, tmp, n, io);
    } else {
        return sort_passes<T, P, 256, 32, 3>(ctx, in, out, tmp, n, io);
    }
}

// ---- split points in a sorted chunk ----------------------------------------------------------------------------------------------------
// counts[i] = number of elements x with NOT (x > bounds[i]) counted from the front of the sorted chunk up to the first x > bounds[i]
// -- i.e. the p_till - 1 of the reference's scan (src/sort.jl:31-38) had it started at element 1: the number of non-NaN elements
// <= bounds[i] (IEEE compare, so -0.0 == +0.0), or n when no element exceeds the bound (NaNs compare false and stay in the piece).
template <typename T>
__global__ void sort_bounds_kernel(const typename SortKey<T>::U* __restrict__ sorted, size_t n, const typename SortKey<T>::U* __restrict__ bounds,
                                   int nb, unsigned long long* __restrict__ counts) {
    using K = SortKey<T>;
    using U = typename K::U;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nb) return;
    U braw = bounds[t];
    bool nan_bound = false;
    if constexpr (sizeof(T) == 4 && !std::is_integral<T>::value) {
        nan_bound = (braw & 0x7FFFFFFFu) > 0x7F800000u;
        if ((braw & 0x7FFFFFFFu) == 0) braw = 0;  // -0.0 bounds like +0.0
    }
    if constexpr (sizeof(T) == 8 && !std::is_integral<T>::value) {
        nan_bound = (braw & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull;
        if ((braw & 0x7FFFFFFFFFFFFFFFull) == 0) braw = 0;
    }
    if (nan_bound) {  // x > NaN is never true
        counts[t] = n;
        return;
    }
    const U kb = K::enc(braw);
    size_t lo = 0, hi = n;  // first index whose key > kb
    while (lo < hi) {
        const size_t mid = lo + ((hi - lo) >> 1);
        if (K::enc(sorted[mid]) <= kb) lo = mid + 1;
        else hi = mid;
    }
    // everything from lo on is either > bound or NaN; if it is all NaN no element exceeds the bound and the scan runs to the end
    bool rest_nan = false;
    if constexpr (!std::is_integral<T>::value) {
        if (lo < n) {
            const U u = sorted[lo];  // smallest remaining key: NaN iff all remaining are NaN (NaNs sort last)
            if constexpr (sizeof(T) == 4) rest_nan = (u & 0x7FFFFFFFu) > 0x7F800000u;
            else rest_nan = (u & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull;
        }
    }
    counts[t] = rest_nan ? n : lo;
}

template <typename T>
int32_t bounds_t(dab_ctx* ctx, const void* sorted, size_t n, const void* bounds_host, int nb, unsigned long long* counts_host) {
    using U = typename SortKey<T>::U;
    DAB_REQUIRE(ctx, nb >= 1 && nb <= 256, DAB_ERR_ARG, "dab_sorted_split: 1..256 bounds");
    int32_t st = sort_scratch(ctx, SORT_PLAN_BYTES);
    if (st != DAB_OK) return st;
    U* dbounds = (U*)((char*)ctx->sort_dev + SORT_PLAN_BYTES - 8192);           // staging behind the SortPlan
    unsigned long long* dcounts = (unsigned long long*)((char*)ctx->sort_dev + SORT_PLAN_BYTES - 4096);
    unsigned long long* hc = (unsigned long long*)((char*)ctx->sort_host + 8 * 256 * sizeof(unsigned long long));
    DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                         // the staging areas may still be in use by a sort
    memcpy(hc, bounds_host, (size_t)nb * sizeof(U));
    DAB_CUDA(ctx, cudaMemcpyAsync(dbounds, hc, (size_t)nb * sizeof(U), cudaMemcpyHostToDevice, ctx->stream));
    sort_bounds_kernel<T><<<(nb + 63) / 64, 64, 0, ctx->stream>>>((const U*)sorted, n, dbounds, nb, dcounts);
    DAB_LAUNCHED(ctx);
    DAB_CUDA(ctx, cudaMemcpyAsync(hc, dcounts, (size_t)nb * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(counts_host, hc, (size_t)nb * sizeof(unsigned long long));
    return DAB_OK;
}

// dab_sort_pairs scratch: the keys' ping-pong buffer, then the two position buffers, each 256-byte aligned
inline size_t pairs_stride(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

inline int pairs_key_bytes(int32_t key_dtype) {
    return (key_dtype == DAB_F64 || key_dtype == DAB_I64) ? 8 : (key_dtype == DAB_F32 || key_dtype == DAB_I32) ? 4 : 0;
}

template <typename T>
int32_t pairs_t(dab_ctx* ctx, const void* keys, void* keys_out, const int64_t* vals, int64_t base, int64_t* vals_out, void* scratch, size_t n) {
    using U = typename SortKey<T>::U;
    char* s = (char*)scratch;
    const size_t ks = pairs_stride(n * sizeof(U)), ps = pairs_stride(n * 4);
    PairIO<uint32_t> io{(uint32_t*)(s + ks), (uint32_t*)(s + ks + ps), vals, base, vals_out};
    return sort_t<T, uint32_t>(ctx, keys, keys_out, s, n, io);
}

}  // namespace

extern "C" {

int32_t dab_sort_pairs_scratch_bytes(int32_t key_dtype, size_t n, size_t* bytes) {
    if (bytes == nullptr) return dab_fail(nullptr, DAB_ERR_ARG, "dab_sort_pairs_scratch_bytes: null pointer");
    const int kb = pairs_key_bytes(key_dtype);
    if (kb == 0) return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "dab_sort_pairs: key dtype %d", key_dtype);
    *bytes = pairs_stride(n * kb) + 2 * pairs_stride(n * 4);
    return DAB_OK;
}

int32_t dab_sort_pairs(dab_ctx* ctx, int32_t key_dtype, const void* keys, void* keys_out, const int64_t* vals, int64_t base, int64_t* vals_out,
                       void* scratch, size_t scratch_bytes, size_t n) {
    DAB_ENTER(ctx);
    if (n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, keys && keys_out && vals_out && scratch, DAB_ERR_ARG, "dab_sort_pairs: null pointer");
    DAB_REQUIRE(ctx, (const void*)vals != (const void*)vals_out, DAB_ERR_ARG, "dab_sort_pairs: vals_out must not alias vals");
    DAB_REQUIRE(ctx, n < 0xFFFFF000ull, DAB_ERR_UNSUPPORTED, "dab_sort_pairs: chunks of 2^32 - 4096 or more elements are not served");
    size_t need = 0;
    int32_t st = dab_sort_pairs_scratch_bytes(key_dtype, n, &need);
    if (st != DAB_OK) return dab_fail(ctx, st, "dab_sort_pairs: key dtype %d", key_dtype);
    DAB_REQUIRE(ctx, scratch_bytes >= need, DAB_ERR_ARG, "dab_sort_pairs: scratch of %zu bytes, %zu needed", scratch_bytes, need);
    DAB_REQUIRE(ctx, ((uintptr_t)scratch & 15) == 0, DAB_ERR_ARG, "dab_sort_pairs: scratch must be 16-byte aligned");
    switch (key_dtype) {
        case DAB_F32: return pairs_t<float>(ctx, keys, keys_out, vals, base, vals_out, scratch, n);
        case DAB_F64: return pairs_t<double>(ctx, keys, keys_out, vals, base, vals_out, scratch, n);
        case DAB_I32: return pairs_t<int32_t>(ctx, keys, keys_out, vals, base, vals_out, scratch, n);
        default: return pairs_t<int64_t>(ctx, keys, keys_out, vals, base, vals_out, scratch, n);
    }
}

int32_t dab_sort(dab_ctx* ctx, int32_t dtype, const void* in, void* out, void* tmp, size_t n) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, n == 0 || (in && out), DAB_ERR_ARG, "dab_sort: null pointer");
    switch (dtype) {
        case DAB_F32: return sort_t<float>(ctx, in, out, tmp, n);
        case DAB_F64: return sort_t<double>(ctx, in, out, tmp, n);
        case DAB_I32: return sort_t<int32_t>(ctx, in, out, tmp, n);
        case DAB_I64: return sort_t<int64_t>(ctx, in, out, tmp, n);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_sort: dtype %d", dtype);
    }
}

int32_t dab_sorted_split(dab_ctx* ctx, int32_t dtype, const void* sorted, size_t n, const void* bounds_host, int32_t nb,
                         unsigned long long* counts_host) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, bounds_host && counts_host && (sorted || n == 0), DAB_ERR_ARG, "dab_sorted_split: null pointer");
    if (n == 0) {
        for (int i = 0; i < nb; ++i) counts_host[i] = 0;
        return DAB_OK;
    }
    switch (dtype) {
        case DAB_F32: return bounds_t<float>(ctx, sorted, n, bounds_host, nb, counts_host);
        case DAB_F64: return bounds_t<double>(ctx, sorted, n, bounds_host, nb, counts_host);
        case DAB_I32: return bounds_t<int32_t>(ctx, sorted, n, bounds_host, nb, counts_host);
        case DAB_I64: return bounds_t<int64_t>(ctx, sorted, n, bounds_host, nb, counts_host);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_sorted_split: dtype %d", dtype);
    }
}

}  // extern "C"
