// lu_host_check.cu -- host-only replay of K27's element code (dab_lu_core.cuh): for every n x n matrix of the input, the path of `A \ b`,
// the pivot sequence of the factorization (a sequential scan with lu_pivot_key / lu_pivot_wins, the order the kernels' reductions
// compute), info of `A \ b`, and det.  Built and run by tests/test_cpu_ldiv.py, which compares with NumPy and SciPy.
//   input:  int64 n, int64 count, then count column-major n x n float64 matrices
//   output: per matrix, float64 [path, info, det, piv_0 .. piv_{n-1}] (piv 0-based, as scipy.linalg.lu_factor)
#include <cstdio>
#include <vector>

#include "dab_lu_core.cuh"

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    FILE* in = fopen(argv[1], "rb");
    FILE* out = fopen(argv[2], "wb");
    if (!in || !out) return 2;
    long long hdr[2];
    if (fread(hdr, sizeof hdr, 1, in) != 1) return 2;
    const int n = (int)hdr[0];
    std::vector<double> a((size_t)n * n);
    for (long long m = 0; m < hdr[1]; ++m) {
        if (fread(a.data(), sizeof(double), a.size(), in) != a.size()) return 2;
        bool nl = false, nu = false, nf = false;
        for (int j = 0; j < n; ++j)
            for (int i = 0; i < n; ++i) {
                nl |= lu_breaks_lower(i, j, a[i + n * j]);
                nu |= lu_breaks_upper(i, j, a[i + n * j]);
                nf |= !std::isfinite(a[i + n * j]);
            }
        const int path = lu_ldiv_path(nl, nu);
        const bool tri = lu_det_triangular(nl, nu);
        std::vector<double> piv(n);
        int swaps = 0, info = 0;
        for (int k = 0; k < n; ++k) {                             // right-looking LU with physical row swaps
            double key = -2.0;
            int p = n;
            for (int i = k; i < n; ++i) {
                const double ki = lu_pivot_key(a[i + n * k], i, k);
                if (lu_pivot_wins(ki, i, key, p)) {
                    key = ki;
                    p = i;
                }
            }
            piv[k] = p;
            if (p != k) {
                ++swaps;
                for (int j = 0; j < n; ++j) std::swap(a[k + n * j], a[p + n * j]);
            }
            const double pv = a[k + n * k];
            if (pv == 0.0) {
                if (info == 0) info = k + 1;
                continue;
            }
            const bool recip = lu_use_reciprocal(pv);
            for (int i = k + 1; i < n; ++i) a[i + n * k] = lu_multiplier(a[i + n * k], pv, 1.0 / pv, recip);
            for (int j = k + 1; j < n; ++j)
                for (int i = k + 1; i < n; ++i) a[i + n * j] = lu_update(a[i + n * j], a[i + n * k], a[k + n * j]);
        }
        // the triangular paths read the diagonal of A itself; the replay re-reads it from the input below when they apply
        double det = 1.0;
        int tinfo = 0;
        if (tri || path != LU_PATH_LU) {
            fseek(in, -(long)(a.size() * sizeof(double)), SEEK_CUR);
            if (fread(a.data(), sizeof(double), a.size(), in) != a.size()) return 2;
            for (int j = 0; j < n; ++j) {
                det = lu_det_step(det, a[j + n * j]);
                if (a[j + n * j] == 0.0 && tinfo == 0) tinfo = j + 1;
            }
        } else {
            for (int j = 0; j < n; ++j) det = lu_det_step(det, a[j + n * j]);
            det = lu_det_finish(det, swaps, info);
        }
        const double ldiv_info = path == LU_PATH_LU ? (nf ? -1.0 : info) : tinfo;
        const double row[3] = {(double)path, ldiv_info, det};
        fwrite(row, sizeof(double), 3, out);
        fwrite(piv.data(), sizeof(double), n, out);
    }
    fclose(in);
    fclose(out);
    printf("lu_host_check: ok\n");
    return 0;
}
