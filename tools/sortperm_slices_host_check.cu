// sortperm_slices_host_check.cu -- host-only replay of K26 (distributedarrays.jl_b200/csrc/dab_sortperm_slices.cu) with the SAME
// per-element code it runs (dab_sortperm_slices_core.cuh).  No GPU, no kernel launch: test infrastructure for the CPU tier
// (tests/test_cpu_sort_dims.py builds and runs it and compares OUT with the stable isless permutation of every fibre).
//   sortperm_slices_host_check PATH IN OUT
//     PATH  net   the pair network of sortperm_slices_kernel: groups of padded fibres in both shapes (inner == 1, inner > 1), the
//                 shared-memory index map, the bitonic directions, the fibre bases and the output places -- for any fibre length
//           long  the long-fibre composition: stable pass by key (K21's order), fibre ids and bases, stable pass by fibre id, finish
//     IN    int64 key_dtype (0 F32, 1 F64, 2 I32, 3 I64), ndim, dim, then chunk_dims[ndim], chunk_lo[ndim], global_dims[ndim], then the
//           n raw keys of the chunk (4 or 8 bytes each, column-major)
//     OUT   the n Int64 entries of perm
//   nvcc -std=c++17 -O2 -I distributedarrays.jl_b200/csrc -I include -o /tmp/sps_check tools/sortperm_slices_host_check.cu
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <vector>

#include "dab200.h"
#include "dab_sortperm_slices_core.cuh"

struct Chunk {
    int ndim, dim;
    size_t dims[DAB_SPS_MAX_DIMS], lo[DAB_SPS_MAX_DIMS], gdims[DAB_SPS_MAX_DIMS];
    size_t inner, len, outer, n;
};

// sortperm_slices_kernel, one group after another, every "thread" of a phase in turn (each phase ends at a __syncthreads)
template <typename T>
static void replay_net(const Chunk& c, const SpsMap& m, const typename SortKey<T>::U* keys, int64_t* perm) {
    using U = typename SortKey<T>::U;
    using SL = SpsSlot<U>;
    const unsigned int CAP = DAB_SORTPERM_SLICES_SMEM_LEN + 64, MAXF = 1024;
    const unsigned int len = (unsigned int)c.len, log2p2 = slices_log2_ceil(c.len), p2 = 1u << log2p2, S = p2 + 1u;
    unsigned int B = CAP / S;
    if (B > MAXF) B = MAXF;
    if (B == 0) B = 1;                                            // fibres longer than the kernel's limit: one per group (replay only)
    std::vector<long long> fb(B);
    std::vector<unsigned long long> w((size_t)B * S, 0x5A5A5A5A5A5A5A5Aull);
    std::vector<unsigned int> ps((size_t)B * S, 0xA5A5A5A5u);
    const size_t ngroups = sps_ngroups(c.inner, c.outer, B);
    for (size_t g = 0; g < ngroups; ++g) {
        const SpsGroup G = sps_group(g, c.inner, len, c.outer, B);
        for (unsigned int t = 0; t < G.nf; ++t) fb[t] = c.inner == 1 ? sps_fibre_base(m, 0, G.o0 + t) : sps_fibre_base(m, G.i0 + t, G.o0);
        for (unsigned int t = 0; t < G.nf * len; ++t) {
            unsigned int b, r;
            const size_t off = sps_group_elem(c.inner, len, G.nf, t, &b, &r);
            w[b * S + r] = SL::word(sortby_radix_key<T>(keys[G.base + off]), r);
            if (SL::SPLIT) ps[b * S + r] = r;
        }
        if (len < p2)
            for (unsigned int t = 0; t < G.nf * p2; ++t) {
                const unsigned int b = t >> log2p2, r = t & (p2 - 1u);
                if (r >= len) {
                    w[b * S + r] = SL::pad();
                    if (SL::SPLIT) ps[b * S + r] = ~0u;
                }
            }
        const unsigned int half = (G.nf * p2) >> 1;
        for (unsigned int k = 2; k <= p2; k <<= 1)
            for (unsigned int j = k >> 1; j > 0; j >>= 1)
                for (unsigned int p = 0; p < half; ++p) {
                    const unsigned int i = slices_bitonic_lo(p, j);
                    const unsigned int ia = slices_smem_index(i, log2p2), ic = slices_smem_index(i + j, log2p2);
                    unsigned int px = SL::SPLIT ? ps[ia] : 0u, py = SL::SPLIT ? ps[ic] : 0u;
                    sps_cmpx<SL::SPLIT>(w[ia], w[ic], px, py, slices_bitonic_asc(i, k, p2));
                    if (SL::SPLIT) ps[ia] = px, ps[ic] = py;
                }
        for (unsigned int t = 0; t < G.nf * len; ++t) {
            unsigned int b, r;
            const size_t off = sps_group_elem(c.inner, len, G.nf, t, &b, &r);
            const unsigned int s = SL::pos(w[b * S + r], SL::SPLIT ? ps[b * S + r] : 0u);
            perm[G.base + off] = fb[b] + (long long)s * (long long)m.gdim;
        }
    }
}

// the long-fibre path: the two K21 passes are stable sorts (by radix key with NaNs collapsed, then by Int32 fibre id) and the two small
// kernels are sortperm_fibre_id_kernel / sortperm_finish_kernel element by element
template <typename T>
static void replay_long(const Chunk& c, const SpsMap& m, const typename SortKey<T>::U* keys, int64_t* perm) {
    const size_t n = c.n;
    std::vector<int64_t> pos1(n), pos2(n);
    std::iota(pos1.begin(), pos1.end(), 0);
    std::stable_sort(pos1.begin(), pos1.end(), [&](int64_t a, int64_t b) { return sortby_radix_key<T>(keys[a]) < sortby_radix_key<T>(keys[b]); });
    std::vector<int32_t> fid(n);
    std::vector<long long> fbase(c.inner * c.outer, -1);
    for (size_t j = 0; j < n; ++j) {
        unsigned int s;
        const unsigned int f = sps_fibre_id((unsigned long long)pos1[j], c.inner, c.len, &s);
        fid[j] = (int32_t)f;
        if (s == 0) {
            unsigned long long i;
            const unsigned long long o = sps_divmod(f, c.inner, &i);
            fbase[f] = sps_fibre_base(m, i, o);
        }
    }
    std::vector<size_t> ord(n);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return fid[a] < fid[b]; });
    for (size_t k = 0; k < n; ++k) pos2[k] = pos1[ord[k]];
    for (size_t k = 0; k < n; ++k) {
        unsigned int s;
        const unsigned int f = sps_fibre_id((unsigned long long)pos2[k], c.inner, c.len, &s);
        perm[sps_out_index(k, c.inner, c.len)] = fbase[f] + (long long)s * (long long)m.gdim;
    }
}

template <typename T>
static void run(bool net, const Chunk& c, const SpsMap& m, const void* keys, int64_t* perm) {
    using U = typename SortKey<T>::U;
    if (net) replay_net<T>(c, m, (const U*)keys, perm);
    else replay_long<T>(c, m, (const U*)keys, perm);
}

int main(int argc, char** argv) {
    if (argc != 4 || (strcmp(argv[1], "net") && strcmp(argv[1], "long"))) {
        std::fprintf(stderr, "usage: %s net|long IN OUT\n", argv[0]);
        return 2;
    }
    const bool net = !strcmp(argv[1], "net");
    FILE* f = std::fopen(argv[2], "rb");
    if (!f) return 2;
    int64_t h[3];
    if (std::fread(h, 8, 3, f) != 3) return 2;
    Chunk c;
    const int dt = (int)h[0];
    c.ndim = (int)h[1];
    c.dim = (int)h[2];
    if (c.ndim < 1 || c.ndim > DAB_SPS_MAX_DIMS) return 2;
    int64_t v[3 * DAB_SPS_MAX_DIMS];
    if (std::fread(v, 8, 3 * c.ndim, f) != (size_t)(3 * c.ndim)) return 2;
    for (int k = 0; k < c.ndim; ++k) c.dims[k] = (size_t)v[k], c.lo[k] = (size_t)v[c.ndim + k], c.gdims[k] = (size_t)v[2 * c.ndim + k];
    SpsMap m;
    if (!sps_make_map(c.ndim, c.dims, c.lo, c.gdims, c.dim, &m)) {
        std::fprintf(stderr, "not a chunk with dimension %d whole\n", c.dim);
        return 3;
    }
    c.inner = c.outer = 1;
    for (int k = 0; k < c.dim - 1; ++k) c.inner *= c.dims[k];
    for (int k = c.dim; k < c.ndim; ++k) c.outer *= c.dims[k];
    c.len = c.dims[c.dim - 1];
    c.n = c.inner * c.len * c.outer;
    const size_t kb = (dt == 1 || dt == 3) ? 8 : 4;
    std::vector<unsigned char> keys(c.n * kb + 8);
    if (std::fread(keys.data(), kb, c.n, f) != c.n) return 2;
    std::fclose(f);
    std::vector<int64_t> perm(c.n, 0);
    switch (dt) {
        case 0: run<float>(net, c, m, keys.data(), perm.data()); break;
        case 1: run<double>(net, c, m, keys.data(), perm.data()); break;
        case 2: run<int32_t>(net, c, m, keys.data(), perm.data()); break;
        case 3: run<int64_t>(net, c, m, keys.data(), perm.data()); break;
        default: return 2;
    }
    FILE* o = std::fopen(argv[3], "wb");
    if (!o || std::fwrite(perm.data(), 8, c.n, o) != c.n) return 2;
    std::fclose(o);
    std::printf("sortperm_slices_host_check: %s %zu elements\n", argv[1], c.n);
    return 0;
}
