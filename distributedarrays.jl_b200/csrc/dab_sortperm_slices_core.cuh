// dab_sortperm_slices_core.cuh -- the per-element arithmetic of K26 (dab_sortperm_slices.cu) as __host__ __device__ functions, so that
// the very same code runs inside the kernels and inside tools/sortperm_slices_host_check.cu (a host-only replay of the pair network and
// of the long-fibre composition against the stable isless permutation; built and run by the CPU test tier).
//
// A chunk is collapsed to (inner, len, outer) around the sorted dimension: fibre (i, o) holds x[i + inner*(s + len*o)], s < len.
#pragma once
#include <cstddef>
#include <cstdint>

#include "dab_slices_core.cuh"
#include "dab_sortby_core.cuh"

constexpr int DAB_SPS_MAX_DIMS = 8;

// ---- global index map -----------------------------------------------------------------------------------------------------------------
// The 1-based global column-major linear index of chunk element x[i + inner*(s + len*o)] is  fibre_base(i, o) + s * gdim  with
//   fibre_base(i, o) = off + sum_k x_k * G_k   over the non-sorted dims k, where (x_k) is i (inner dims) or o (outer dims) in mixed radix
//   off = 1 + sum_k chunk_lo[k] * G_k,  G_k = prod(global_dims[0:k]),  gdim = G_{dim-1}.
struct SpsMap {
    unsigned long long off, gdim;
    int nin, nout;                                  // non-sorted dims before / after the sorted one
    unsigned long long ext_in[DAB_SPS_MAX_DIMS - 1], g_in[DAB_SPS_MAX_DIMS - 1];     // chunk extents and global strides G_k, inner dims
    unsigned long long ext_out[DAB_SPS_MAX_DIMS - 1], g_out[DAB_SPS_MAX_DIMS - 1];   // ... outer dims (fixed slots: no dynamic indexing)
};

// false when the description is not a chunk whose dimension `dim` (1-based) is whole
__host__ __device__ inline bool sps_make_map(int ndim, const size_t* chunk_dims, const size_t* chunk_lo, const size_t* global_dims, int dim,
                                             SpsMap* m) {
    if (ndim < 1 || ndim > DAB_SPS_MAX_DIMS || dim < 1 || dim > ndim) return false;
    unsigned long long G = 1;
    m->off = 1;
    m->nin = m->nout = 0;
    for (int j = 0; j < DAB_SPS_MAX_DIMS - 1; ++j) m->ext_in[j] = m->ext_out[j] = 1, m->g_in[j] = m->g_out[j] = 0;
    for (int k = 0; k < ndim; ++k) {
        if (chunk_lo[k] + chunk_dims[k] > global_dims[k]) return false;
        m->off += (unsigned long long)chunk_lo[k] * G;
        if (k == dim - 1) {
            if (chunk_dims[k] != global_dims[k]) return false;
            m->gdim = G;
        } else if (k < dim - 1) {
            m->ext_in[m->nin] = chunk_dims[k];
            m->g_in[m->nin++] = G;
        } else {
            m->ext_out[m->nout] = chunk_dims[k];
            m->g_out[m->nout++] = G;
        }
        G *= (unsigned long long)global_dims[k];
    }
    return true;
}

// x / d and x % d with the 32-bit divide when both fit (the common case; the 64-bit divide is a long subroutine)
__host__ __device__ inline unsigned long long sps_divmod(unsigned long long x, unsigned long long d, unsigned long long* rem) {
    unsigned long long q;
    if ((x | d) >> 32) q = x / d;
    else q = (unsigned int)x / (unsigned int)d;
    *rem = x - q * d;
    return q;
}

__host__ __device__ inline long long sps_fibre_base(const SpsMap& m, unsigned long long i, unsigned long long o) {
    unsigned long long b = m.off, r;                            // fixed trip counts: the loops unroll, m stays in registers
    for (int k = 0; k < DAB_SPS_MAX_DIMS - 1; ++k)
        if (k < m.nin) {
            i = sps_divmod(i, m.ext_in[k], &r);
            b += r * m.g_in[k];
        }
    for (int k = 0; k < DAB_SPS_MAX_DIMS - 1; ++k)
        if (k < m.nout) {
            o = sps_divmod(o, m.ext_out[k], &r);
            b += r * m.g_out[k];
        }
    return (long long)b;
}

// ---- short fibres: the pair network --------------------------------------------------------------------------------------------------
// A slot is (radix key, position s in the fibre), compared lexicographically.  The radix key is sortby_radix_key (every NaN collapsed to
// the top key, so NaNs are ties); positions are unique within a fibre, so the slot order is a strict total order and the bitonic network
// (unstable in general) yields exactly the stable isless order.  32-bit keys pack into one word key << 32 | s; 64-bit keys keep the
// position in a parallel array.  The pad slot (all ones, all ones) is above every real slot: a real position is < len <= 2^32 - 1.
template <typename U> struct SpsSlot;
template <> struct SpsSlot<uint32_t> {
    using W = unsigned long long;                   // the word compared by the network
    static constexpr bool SPLIT = false;            // no position array
    __host__ __device__ static W word(uint32_t key, unsigned int s) { return ((W)key << 32) | s; }
    __host__ __device__ static unsigned int pos(W w, unsigned int) { return (unsigned int)w; }
    __host__ __device__ static W pad() { return ~(W)0; }
};
template <> struct SpsSlot<uint64_t> {
    using W = unsigned long long;
    static constexpr bool SPLIT = true;
    __host__ __device__ static W word(uint64_t key, unsigned int) { return key; }
    __host__ __device__ static unsigned int pos(W, unsigned int p) { return p; }
    __host__ __device__ static W pad() { return ~(W)0; }
};

// compare/exchange of slots a < b of a bitonic stage (pa / pb: the positions of SPLIT slots, unused otherwise)
template <bool SPLIT>
__host__ __device__ inline void sps_cmpx(unsigned long long& a, unsigned long long& b, unsigned int& pa, unsigned int& pb, bool asc) {
    const bool gt = SPLIT ? (a > b || (a == b && pa > pb)) : a > b;
    if (gt == asc) {
        const unsigned long long t = a;
        a = b;
        b = t;
        if (SPLIT) {
            const unsigned int u = pa;
            pa = pb;
            pb = u;
        }
    }
}

// Group geometry, the same as dab_sort_slices: B fibres of P2 = 2^log2p2 slots, at most SPS_MAX_FIBRES of them.
//   inner == 1: group g is fibres o0 = g*B .. o0 + nf - 1, one contiguous run of nf * len elements starting at `base`;
//   inner  > 1: group g is fibres i0 = (g mod gpo)*B .. i0 + nf - 1 of one o: row r is the nf contiguous elements base + r*inner + b.
struct SpsGroup {
    size_t base, i0, o0;
    unsigned int nf;
};
__host__ __device__ inline SpsGroup sps_group(size_t g, size_t inner, unsigned int len, size_t outer, unsigned int B) {
    SpsGroup G;
    if (inner == 1) {
        G.i0 = 0;
        G.o0 = g * B;
        G.nf = (unsigned int)(outer - G.o0 < B ? outer - G.o0 : B);
        G.base = G.o0 * len;
    } else {
        const size_t gpo = (inner + B - 1) / B;
        G.o0 = g / gpo;
        G.i0 = (g - G.o0 * gpo) * B;
        G.nf = (unsigned int)(inner - G.i0 < B ? inner - G.i0 : B);
        G.base = G.o0 * inner * len + G.i0;
    }
    return G;
}
__host__ __device__ inline size_t sps_ngroups(size_t inner, size_t outer, unsigned int B) {
    return inner == 1 ? (outer + B - 1) / B : ((inner + B - 1) / B) * outer;
}
// element t < nf * len of a group -> (fibre b, position r) and its chunk offset from the group's base (loads and stores alike)
__host__ __device__ inline size_t sps_group_elem(size_t inner, unsigned int len, unsigned int nf, unsigned int t, unsigned int* b,
                                                 unsigned int* r) {
    if (inner == 1) {
        *b = t / len;
        *r = t - *b * len;
        return t;
    }
    *r = t / nf;
    *b = t - *r * nf;
    return (size_t)*r * inner + *b;
}
// chunk offset of position s of fibre b, from the group's base
__host__ __device__ inline size_t sps_group_offset(size_t inner, unsigned int len, unsigned int b, unsigned int s) {
    return inner == 1 ? (size_t)b * len + s : (size_t)s * inner + b;
}

// ---- long fibres: two chunk-wide stable pair sorts (K21) -----------------------------------------------------------------------------
// Pass 1 orders the chunk positions q by key.  Every q then gets its fibre id f = (q mod inner) + inner * (q div (inner*len)) = i + inner*o,
// and pass 2 orders the positions by fibre id, stably: fibre-major, key order inside each fibre.  Entry k of that order is rank
// r = k mod len of fibre f = k div len, written at i + inner*(r + len*o).  Fibre ids are below n / len < 2^32 / DAB_SORTPERM_SLICES_SMEM_LEN,
// so they are Int32 keys.
__host__ __device__ inline unsigned int sps_fibre_id(unsigned long long q, unsigned long long inner, unsigned long long len, unsigned int* s) {
    unsigned long long i, sl;
    const unsigned long long c = sps_divmod(q, inner, &i);      // s + len*o
    const unsigned long long o = sps_divmod(c, len, &sl);
    *s = (unsigned int)sl;
    return (unsigned int)(i + inner * o);
}
// output place of entry k of the fibre-major order
__host__ __device__ inline size_t sps_out_index(unsigned long long k, unsigned long long inner, unsigned long long len) {
    unsigned long long r, i;
    const unsigned long long f = sps_divmod(k, len, &r);
    const unsigned long long o = sps_divmod(f, inner, &i);
    return (size_t)(i + inner * (r + len * o));
}
