// onepass_emu.cpp — runs the SOURCE of the one-pass dense GKL kernels (krylovkit.jl_b200/csrc/onepass_kernels.cuh)
// on host threads through tests/emu/cuda_emu.h and checks y = A x, z = A'(A x) against plain double loops, for the
// launch geometries the host code of spmv.cu uses (variant A: 256 threads, NZ by width; variant B: 512 threads;
// then k_onepass_reduce).  Test infrastructure: built by tests/test_onepass_emulation.py with g++ and a sanitizer,
// and without one for the dump mode below, which the summation-order restatement is compared with.
#define B2K_HOST_EMU 1
#include "cuda_emu.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>

namespace {
#include "onepass_kernels.cuh"
}

template <typename T>
static int run_case(int64_t m, int n, int grid_cap, int variant) {
    const int64_t ld = (m + 31) / 32 * 32;
    std::mt19937_64 rng(1234 + m * 7 + n);
    std::uniform_real_distribution<double> U(-0.5, 0.5);
    T* A = new T[(size_t)ld * n];                    // exact size: an out-of-range load is an ASan error
    for (int c = 0; c < n; ++c)
        for (int64_t i = 0; i < ld; ++i) A[(size_t)c * ld + i] = i < m ? (T)U(rng) : (T)0;
    T* x = new T[n];
    for (int c = 0; c < n; ++c) x[c] = (T)U(rng);
    T* y = new T[m];
    T* z = new T[n];
    for (int64_t i = 0; i < m; ++i) y[i] = (T)1e30;
    int grid = 0;
    double* zpart = nullptr;
    if (variant == 0) {
        const int64_t ntiles = ld / OP_ROWS;
        grid = (int)std::min<int64_t>(ntiles, grid_cap);
        zpart = new double[(size_t)grid * n];
        const size_t smem = ((size_t)n * OP_PAD + n + (OP_T / 32) * OP_ROWS + OP_ROWS) * sizeof(T);
        auto call = [&]() {
            if (n <= OP_T) k_dense_onepass<T, 1>(A, ld, m, n, x, y, zpart, ntiles);
            else if (n <= 2 * OP_T) k_dense_onepass<T, 2>(A, ld, m, n, x, y, zpart, ntiles);
            else if (n <= 4 * OP_T) k_dense_onepass<T, 4>(A, ld, m, n, x, y, zpart, ntiles);
            else k_dense_onepass<T, OP_ZMAX>(A, ld, m, n, x, y, zpart, ntiles);
        };
        b2k_emu::launch(grid, OP_T, smem, call);
    } else {
        if constexpr (sizeof(T) == 4) {
            const int64_t ntiles = (ld + OPW_ROWS - 1) / OPW_ROWS;
            grid = (int)std::min<int64_t>(ntiles, grid_cap);
            zpart = new double[(size_t)grid * n];
            const size_t smem = ((size_t)n * OPW_PAD + n + (OPW_T / 32) * OPW_ROWS + OPW_ROWS) * sizeof(float);
            b2k_emu::launch(grid, OPW_T, smem, [&]() { k_dense_onepass_w(A, ld, m, n, x, y, zpart, ntiles); });
        }
    }
    double* dres = new double[n];
    b2k_emu::launch((n + 31) / 32, 256, 0, [&]() { k_onepass_reduce<T>(zpart, grid, n, dres, z); });
    // reference
    int bad = 0;
    const double eps = sizeof(T) == 4 ? 1.2e-7 : 2.3e-16;
    std::vector<double> yr(m, 0.0), zr(n, 0.0);
    double ymax = 0, zmax = 0;
    for (int64_t i = 0; i < m; ++i) {
        double s = 0;
        for (int c = 0; c < n; ++c) s += (double)A[(size_t)c * ld + i] * (double)x[c];
        yr[i] = s;
        ymax = std::max(ymax, std::fabs(s));
    }
    for (int c = 0; c < n; ++c) {
        double s = 0;
        for (int64_t i = 0; i < m; ++i) s += (double)A[(size_t)c * ld + i] * (double)y[i];     // A' of the y that was formed
        zr[c] = s;
        zmax = std::max(zmax, std::fabs(s));
    }
    for (int64_t i = 0; i < m; ++i)
        if (!(std::fabs((double)y[i] - yr[i]) <= 16 * eps * std::sqrt((double)n) * ymax + 1e-300)) ++bad;
    for (int c = 0; c < n; ++c) {
        if (!(std::fabs((double)z[c] - zr[c]) <= 16 * eps * std::sqrt((double)m) * zmax + 1e-300)) ++bad;
        if (!(std::fabs(dres[c] - zr[c]) <= 16 * eps * std::sqrt((double)m) * zmax + 1e-300)) ++bad;
    }
    std::printf("%s m=%lld n=%d %s grid=%d variant=%c\n", bad ? "FAIL" : "ok", (long long)m, n, sizeof(T) == 4 ? "f32" : "f64",
                grid, variant ? 'B' : 'A');
    delete[] A; delete[] x; delete[] y; delete[] z; delete[] zpart; delete[] dres;
    return bad;
}

// `onepass_emu dump IN OUT`: one launch of the kernels on the data of IN, every output written to OUT, so that
// oracle/onepass_restate.py can be compared with the kernel source bit for bit (test_onepass_emulation.py).
//   IN : int32 dtype size (4 / 8), int32 variant (0 = A, 1 = B), int64 m, int32 n, int32 grid,
//        A (ld x n column-major in T, ld = 32 ceil(m / 32), rows [m, ld) zero), x (n, T)
//   OUT: y (m, T), zpart (grid x n doubles), dres (n doubles), z (n, T)
template <typename T>
static int dump_case(std::FILE* in, std::FILE* out, int variant, int64_t m, int n, int grid) {
    const int64_t ld = (m + 31) / 32 * 32;
    std::vector<T> A((size_t)ld * n), x(n), y(m, (T)1e30), z(n);
    std::vector<double> zpart((size_t)grid * n, 0.0), dres(n);
    if (std::fread(A.data(), sizeof(T), A.size(), in) != A.size() || std::fread(x.data(), sizeof(T), n, in) != (size_t)n)
        return 2;
    if (variant == 0) {
        const int64_t ntiles = ld / OP_ROWS;
        if (grid < 1 || grid > ntiles) return 3;
        const size_t smem = ((size_t)n * OP_PAD + n + (OP_T / 32) * OP_ROWS + OP_ROWS) * sizeof(T);
        b2k_emu::launch(grid, OP_T, smem, [&]() {
            if (n <= OP_T) k_dense_onepass<T, 1>(A.data(), ld, m, n, x.data(), y.data(), zpart.data(), ntiles);
            else if (n <= 2 * OP_T) k_dense_onepass<T, 2>(A.data(), ld, m, n, x.data(), y.data(), zpart.data(), ntiles);
            else if (n <= 4 * OP_T) k_dense_onepass<T, 4>(A.data(), ld, m, n, x.data(), y.data(), zpart.data(), ntiles);
            else k_dense_onepass<T, OP_ZMAX>(A.data(), ld, m, n, x.data(), y.data(), zpart.data(), ntiles);
        });
    } else {
        if constexpr (sizeof(T) == 4) {
            const int64_t ntiles = (ld + OPW_ROWS - 1) / OPW_ROWS;
            if (grid < 1 || grid > ntiles || n > 512) return 3;
            const size_t smem = ((size_t)n * OPW_PAD + n + (OPW_T / 32) * OPW_ROWS + OPW_ROWS) * sizeof(float);
            b2k_emu::launch(grid, OPW_T, smem, [&]() {
                k_dense_onepass_w(A.data(), ld, m, n, x.data(), y.data(), zpart.data(), ntiles);
            });
        } else {
            return 3;
        }
    }
    b2k_emu::launch((n + 31) / 32, 256, 0, [&]() { k_onepass_reduce<T>(zpart.data(), grid, n, dres.data(), z.data()); });
    std::fwrite(y.data(), sizeof(T), m, out);
    std::fwrite(zpart.data(), sizeof(double), zpart.size(), out);
    std::fwrite(dres.data(), sizeof(double), n, out);
    std::fwrite(z.data(), sizeof(T), n, out);
    return 0;
}

static int dump(const char* inpath, const char* outpath) {
    std::FILE* in = std::fopen(inpath, "rb");
    if (!in) return 2;
    int32_t tsize = 0, variant = 0, n = 0, grid = 0;
    int64_t m = 0;
    if (std::fread(&tsize, 4, 1, in) != 1 || std::fread(&variant, 4, 1, in) != 1 || std::fread(&m, 8, 1, in) != 1 ||
        std::fread(&n, 4, 1, in) != 1 || std::fread(&grid, 4, 1, in) != 1 || m < 1 || n < 1) {
        std::fclose(in);
        return 2;
    }
    std::FILE* out = std::fopen(outpath, "wb");
    if (!out) {
        std::fclose(in);
        return 2;
    }
    const int rc = tsize == 4 ? dump_case<float>(in, out, variant, m, n, grid)
                 : tsize == 8 ? dump_case<double>(in, out, variant, m, n, grid) : 2;
    std::fclose(in);
    if (std::fclose(out) != 0) return 2;
    return rc;
}

int main(int argc, char** argv) {
    if (argc == 4 && std::string(argv[1]) == "dump") return dump(argv[2], argv[3]);
    const bool quick = argc > 1 && std::atoi(argv[1]) == 1;
    int bad = 0;
    if (argc > 1 && std::atoi(argv[1]) == 2) {          // a longer run by hand: many tiles per CTA at config 4's width
        bad += run_case<float>(3000, 512, 4, 0);
        bad += run_case<float>(3000, 512, 3, 1);
        bad += run_case<float>(3040, 512, 1, 1);        // ld = 3040 = 47.5 tiles of 64 rows, one CTA walks them all
        bad += run_case<float>(3040, 512, 7, 0);
        std::printf(bad ? "FAILED\n" : "all ok\n");
        return bad ? 1 : 0;
    }
    bad += run_case<float>(100, 70, 3, 0);
    bad += run_case<float>(100, 70, 2, 1);
    bad += run_case<float>(96, 300, 2, 1);          // ld = 96: the last 64-row tile of variant B is half outside A
    bad += run_case<double>(70, 40, 2, 0);
    if (!quick) {
        bad += run_case<float>(257, 512, 3, 0);
        bad += run_case<float>(160, 512, 2, 1);
        bad += run_case<float>(33, 600, 1, 0);      // NZ = 4
        bad += run_case<float>(64, 1100, 1, 0);     // NZ = 7
        bad += run_case<double>(130, 300, 2, 0);    // NZ = 2, double2 loads
        bad += run_case<float>(4000, 6, 5, 0);
        bad += run_case<float>(4000, 6, 5, 1);
    }
    std::printf(bad ? "FAILED\n" : "all ok\n");
    return bad ? 1 : 0;
}
