// ppeval_host_check.cu -- host-only replay of eigvals_sym_kernel (distributedarrays.jl_b200/csrc/dab_batched.cu) with the SAME per-element
// code it runs (dab_slices_core.cuh): scaling, round-robin pairs, rotations, convergence test, ranking.  No GPU, no kernel launch: test
// infrastructure for the CPU tier (tests/test_cpu_ppeval.py builds and runs it against numpy.linalg.eigvalsh).
//   ppeval_host_check IN OUT   IN holds int64 n, batch and then the batch column-major fp64 n x n matrices; OUT receives, per matrix, the
//                              n eigenvalues ascending followed by the number of sweeps the kernel would run (as a double)
//   nvcc -std=c++17 -O2 -I distributedarrays.jl_b200/csrc -o /tmp/ppeval_host_check tools/ppeval_host_check.cu
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "dab_slices_core.cuh"

// one matrix, round by round in the kernel's order: every rotation of the round from the current pivots, then all rows, then all columns,
// then the rotated off-diagonal pairs set to 0
static int replay(std::vector<double>& M, int n, std::vector<double>& w) {
    double amax = 0.0;
    for (double v : M) amax = std::fmax(amax, std::fabs(v));
    const int e = slices_scale_exp(amax);
    for (double& v : M) v = std::ldexp(v, -e);
    const int np = n + (n & 1), npairs = np / 2;
    std::vector<double> cs(npairs), sn(npairs);
    int sweeps = 0;
    for (int sweep = 0; sweep < DAB_EIG_MAX_SWEEPS; ++sweep) {
        ++sweeps;
        bool rot = false;
        for (int r = 0; r < np - 1; ++r) {
            for (int k = 0; k < npairs; ++k) {
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                double c = 1.0, s = 0.0;
                if (p < n && q < n && slices_sym_rotation(M[p + n * p], M[q + n * q], M[p + n * q], &c, &s)) rot = true;
                cs[k] = c;
                sn[k] = s;
            }
            for (int k = 0; k < npairs; ++k) {
                if (sn[k] == 0.0) continue;
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                for (int j = 0; j < n; ++j) slices_jacobi_apply(&M[p + n * j], &M[q + n * j], cs[k], sn[k]);
            }
            for (int k = 0; k < npairs; ++k) {
                if (sn[k] == 0.0) continue;
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                for (int i = 0; i < n; ++i) slices_jacobi_apply(&M[i + n * p], &M[i + n * q], cs[k], sn[k]);
            }
            for (int k = 0; k < npairs; ++k) {
                if (sn[k] == 0.0) continue;
                int p, q;
                slices_rr_pair(np, r, k, &p, &q);
                M[p + n * q] = 0.0;
                M[q + n * p] = 0.0;
            }
        }
        if (!rot) break;
    }
    std::vector<double> d(n);
    for (int t = 0; t < n; ++t) d[t] = M[t + n * t];
    w.assign(n, 0.0);
    for (int t = 0; t < n; ++t) w[slices_rank_asc(d.data(), n, t)] = std::ldexp(d[t], e);
    return sweeps;
}

int main(int argc, char** argv) {
    if (argc != 3) {
        std::fprintf(stderr, "usage: ppeval_host_check IN OUT\n");
        return 2;
    }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    int64_t hdr[2];
    if (std::fread(hdr, sizeof(int64_t), 2, f) != 2) return 2;
    const int n = (int)hdr[0];
    const int64_t batch = hdr[1];
    if (n < 1 || n > 64) {
        std::fprintf(stderr, "n = %d outside 1..64\n", n);
        return 2;
    }
    FILE* g = std::fopen(argv[2], "wb");
    if (!g) return 2;
    std::vector<double> M((size_t)n * n), w;
    for (int64_t b = 0; b < batch; ++b) {
        if (std::fread(M.data(), sizeof(double), M.size(), f) != M.size()) return 2;
        const double sweeps = replay(M, n, w);
        std::fwrite(w.data(), sizeof(double), n, g);
        std::fwrite(&sweeps, sizeof(double), 1, g);
    }
    std::fclose(f);
    std::fclose(g);
    std::printf("ppeval_host_check: ok\n");
    return 0;
}
