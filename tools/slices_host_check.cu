// slices_host_check.cu -- host-only replay of the slice kernels (distributedarrays.jl_b200/csrc/dab_slices.cu) with the SAME per-element
// code they run (dab_slices_core.cuh).  No GPU, no kernel launch: test infrastructure for the CPU tier (tests/test_cpu_mapslices.py builds
// and runs it).
//   slices_host_check              the bitonic network of sort_slices_kernel (groups of padded fibres, shared-memory index map, directions)
//                                  against std::sort of the encoded keys, for the four dtypes; exit code 0 = every fibre identical
//   slices_host_check svd IN OUT   the Jacobi sweeps of svdvals_kernel, serialised round by round: IN holds int64 m, n, batch and then
//                                  the batch column-major fp64 matrices; OUT receives the k = min(m, n) values of each, descending
//   nvcc -std=c++17 -O2 -I distributedarrays.jl_b200/csrc -o /tmp/slices_host_check tools/slices_host_check.cu
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <random>
#include <vector>

#include "dab_slices_core.cuh"

// one CTA's group: nf fibres of len keys, padded to P2, sorted by the kernel's network
template <typename T>
static std::vector<typename SortKey<T>::U> replay_group(const std::vector<typename SortKey<T>::U>& raw, unsigned int nf, unsigned int len) {
    using K = SortKey<T>;
    using U = typename K::U;
    const unsigned int log2p2 = slices_log2_ceil(len), p2 = 1u << log2p2;
    std::vector<U> s((size_t)nf * (p2 + 1), (U)0x5A);
    for (unsigned int b = 0; b < nf; ++b)
        for (unsigned int r = 0; r < p2; ++r) s[b * (p2 + 1) + r] = r < len ? K::enc(raw[(size_t)b * len + r]) : slices_pad_key<U>();
    const unsigned int half = (nf * p2) >> 1;
    for (unsigned int k = 2; k <= p2; k <<= 1)
        for (unsigned int j = k >> 1; j > 0; j >>= 1)
            for (unsigned int p = 0; p < half; ++p) {
                const unsigned int i = slices_bitonic_lo(p, j);
                slices_cmpx(s[slices_smem_index(i, log2p2)], s[slices_smem_index(i + j, log2p2)], slices_bitonic_asc(i, k, p2));
            }
    std::vector<U> out((size_t)nf * len);
    for (unsigned int b = 0; b < nf; ++b)
        for (unsigned int r = 0; r < len; ++r) out[(size_t)b * len + r] = K::dec(s[b * (p2 + 1) + r]);
    return out;
}

template <typename T>
static int check_sort(const char* name, std::mt19937_64& rng) {
    using K = SortKey<T>;
    using U = typename K::U;
    int bad = 0;
    for (unsigned int len : {1u, 2u, 5u, 31u, 32u, 33u, 100u, 1000u, 4096u, 4097u, 8192u})
        for (unsigned int nf : {1u, 3u, 8u}) {
            std::vector<U> raw((size_t)nf * len);
            for (auto& v : raw) v = (U)rng();
            if constexpr (std::is_floating_point<T>::value) {   // signed zeros, infinities, NaNs of both signs and several payloads
                const uint32_t special4[] = {0x00000000u, 0x80000000u, 0x7F800000u, 0xFF800000u, 0x7FC00000u, 0xFFC00001u, 0x7F800123u, 0x3F800000u};
                const uint64_t special8[] = {0ull, 0x8000000000000000ull, 0x7FF0000000000000ull, 0xFFF0000000000000ull, 0x7FF8000000000000ull,
                                      0xFFF8000000000001ull, 0x7FF0000000000123ull, 0x3FF0000000000000ull};
                for (size_t t = 0; t < raw.size() / 3 + 1; ++t)
                    raw[rng() % raw.size()] = sizeof(U) == 4 ? (U)special4[rng() % 8] : (U)special8[rng() % 8];
            } else if (raw.size() > 4) {   // integer extremes
                raw[0] = (U)std::numeric_limits<T>::min();
                raw[1] = (U)std::numeric_limits<T>::max();
                raw[2] = (U)~(U)0;   // -1, whose key is NOT all ones; an all-ones key (typemax) is above
            }
            const std::vector<U> got = replay_group<T>(raw, nf, len);
            for (unsigned int b = 0; b < nf; ++b) {
                std::vector<U> want(raw.begin() + (size_t)b * len, raw.begin() + (size_t)(b + 1) * len);
                for (auto& v : want) v = K::enc(v);
                std::sort(want.begin(), want.end());
                for (auto& v : want) v = K::dec(v);
                if (!std::equal(want.begin(), want.end(), got.begin() + (size_t)b * len)) {
                    std::printf("FAIL %s len=%u nf=%u fibre %u\n", name, len, nf, b);
                    ++bad;
                }
            }
        }
    return bad;
}

// svdvals_kernel with the rounds serialised: the pairs of one round touch disjoint columns, so running them one after the other gives
// the same arithmetic as the warps running them at once (each dot product is summed here in row order instead of by lane + shuffle)
static std::vector<double> replay_svd(const double* a, int m, int n) {
    const bool tr = n > m;
    const int M = tr ? n : m, nc = tr ? m : n, np = nc + (nc & 1);
    std::vector<double> W((size_t)M * nc);
    double amax = 0.0;
    for (int t = 0; t < m * n; ++t) {
        const int row = t % m, col = t / m;
        W[tr ? col + M * row : t] = a[t];
        amax = std::fmax(amax, std::fabs(a[t]));
    }
    const int e = slices_scale_exp(amax);
    for (auto& w : W) w = std::ldexp(w, -e);
    const double tol = slices_jacobi_tol(M);
    for (int sweep = 0; sweep < DAB_SVD_MAX_SWEEPS; ++sweep) {
        bool rot = false;
        for (int r = 0; r < np - 1; ++r)
            for (int k = 0; k < np / 2; ++k) {
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                if (p >= nc || q >= nc) continue;
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < M; ++i) {
                    const double x = W[i + M * p], y = W[i + M * q];
                    al += x * x;
                    be += y * y;
                    ga += x * y;
                }
                double c, s;
                if (slices_jacobi_rotation(al, be, ga, tol, &c, &s)) {
                    rot = true;
                    for (int i = 0; i < M; ++i) slices_jacobi_apply(&W[i + M * p], &W[i + M * q], c, s);
                }
            }
        if (!rot) break;
    }
    std::vector<double> sv(nc);
    for (int c = 0; c < nc; ++c) {
        double ss = 0;
        for (int i = 0; i < M; ++i) ss += W[i + M * c] * W[i + M * c];
        sv[c] = std::ldexp(std::sqrt(ss), e);
    }
    std::sort(sv.begin(), sv.end(), [](double x, double y) { return x > y; });
    return sv;
}

static int run_svd(const char* in_path, const char* out_path) {
    FILE* f = std::fopen(in_path, "rb");
    if (!f) return 2;
    int64_t hdr[3];
    if (std::fread(hdr, 8, 3, f) != 3) return 2;
    const int m = (int)hdr[0], n = (int)hdr[1];
    const size_t batch = (size_t)hdr[2], mn = (size_t)m * n;
    std::vector<double> a(mn * batch);
    if (std::fread(a.data(), 8, a.size(), f) != a.size()) return 2;
    std::fclose(f);
    std::vector<double> out;
    for (size_t b = 0; b < batch; ++b) {
        const std::vector<double> sv = replay_svd(a.data() + b * mn, m, n);
        out.insert(out.end(), sv.begin(), sv.end());
    }
    FILE* g = std::fopen(out_path, "wb");
    if (!g) return 2;
    std::fwrite(out.data(), 8, out.size(), g);
    std::fclose(g);
    return 0;
}

int main(int argc, char** argv) {
    if (argc == 4 && std::strcmp(argv[1], "svd") == 0) return run_svd(argv[2], argv[3]);
    std::mt19937_64 rng(20261015);
    int bad = check_sort<float>("Float32", rng) + check_sort<double>("Float64", rng) + check_sort<int32_t>("Int32", rng) +
              check_sort<int64_t>("Int64", rng);
    // round-robin pairing: every pair of columns exactly once per sweep, the pairs of a round disjoint
    for (int np = 2; np <= 32; np += 2) {
        std::vector<int> seen(np * np, 0);
        for (int r = 0; r < np - 1; ++r) {
            std::vector<int> used(np, 0);
            for (int k = 0; k < np / 2; ++k) {
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                if (p == q || used[p]++ || used[q]++) { std::printf("FAIL pairing np=%d round %d\n", np, r); ++bad; }
                ++seen[std::min(p, q) * np + std::max(p, q)];
            }
        }
        for (int p = 0; p < np; ++p)
            for (int q = p + 1; q < np; ++q)
                if (seen[p * np + q] != 1) { std::printf("FAIL pairing np=%d pair (%d,%d)\n", np, p, q); ++bad; }
    }
    std::printf(bad ? "slices_host_check: %d FAILED\n" : "slices_host_check: ok\n", bad);
    return bad ? 1 : 0;
}
