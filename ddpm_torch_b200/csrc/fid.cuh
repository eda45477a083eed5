// Fréchet Inception Distance (ddpm_torch/metrics/fid_score.py): streaming fp64 feature statistics and the Fréchet distance.
// The reference copies every batch of Inception features to the host for np.cov and a Chan merge (:116-135), and takes
// scipy.linalg.sqrtm of the non-symmetric product sigma1 . sigma2 by a complex Schur decomposition (:269-323).
//
// Statistics.  The caller-owned state holds a shift c[D] (the column means of the first non-empty batch, fixed-order sums), the
// shifted sum s[D] = sum (x - c) and the shifted co-moment Cm = sum (x - c)^T (x - c) (lower-triangle 64 x 64 tiles only); the row
// count n stays on the host.  mean = c + s / n and cov = (Cm - s s^T / n) / (n - ddof).  The co-moment is a DMMA (fp64 tensor core,
// mma.sync m16n8k4) GEMM in which each CTA owns one output tile and walks every row of the batch: no atomics, so two runs on the same
// batches are bit-identical.  fp32 x fp32 products are exact in fp64, so this is np.cov's fp64 arithmetic up to reordering.
//
// Distance.  ||mu1 - mu2||^2 + tr S1 + tr S2 - 2 tr sqrt(S1 S2) by a real, symmetric route: with S1 = Q diag(lam) Q^T and
// L = Q diag(sqrt(max(lam, 0))), the eigenvalues of S1 S2 are those of the PSD matrix M = L^T S2 L, so tr sqrt(S1 S2) = sum sqrt(nu).
// Both eigen-solves are one-sided (Hestenes) Jacobi with parallel round-robin ordering, run by one cooperative kernel that rotates
// D/2 disjoint row pairs per round and synchronises the grid between rounds; a sweep without a rotation ends it, and a hard cap on
// sweeps returns an error code.  The rows of W = A V converge to lam_i v_i, so lam_i = sign(v_i . w_i) ||w_i||: V is accumulated
// for M as well, because that sign is how a non-PSD S2 shows.  M is L^T (S2 L), two DMMA GEMMs.  Every reduction runs in a fixed order.
#pragma once
#include <cooperative_groups.h>
#include "ptx.cuh"

namespace ddpm {

constexpr int FID_MAX_D = 4096;
constexpr int FID_TILE = 64;                     // GEMM output tile; D is zero-padded to a multiple of it
constexpr int FID_KC = 16;                       // batch rows per shared-memory chunk of the GEMM
constexpr int FID_SPAD = FID_TILE + 4;           // row pitch (doubles) of the GEMM's shared tiles: conflict-free fragment loads
constexpr int FID_MAX_SWEEPS = 60;
constexpr double FID_NEG_TOL = 1e-6;             // lam_min < -FID_NEG_TOL * lam_max: not PSD beyond rounding
constexpr size_t FID_HDR = 256;

// ddpm_fid_distance's status (out[1]) and the error codes of its entry point
enum FidStatus { FID_OK = 0, FID_NONFINITE = 1, FID_NOT_PSD_1 = 2, FID_NOT_PSD_M = 3, FID_NO_CONV_1 = 4, FID_NO_CONV_M = 5 };

inline int fid_pad(int D) { return (D + FID_TILE - 1) / FID_TILE * FID_TILE; }
inline size_t fid_al(size_t b) { return (b + 255) & ~size_t(255); }
// state: header (i32 initialised) | c f64[Dp] | s f64[Dp] | Cm f64[Dp][Dp]
inline size_t fid_stats_bytes(int D) { const size_t p = fid_pad(D); return FID_HDR + fid_al(p * 8) * 2 + fid_al(p * p * 8); }
// scratch: header (status, 2 x 3 sweep counters, 2 sweep counts) | lam f64[Dp] | nu f64[Dp] | W, V, S2, L f64[Dp][Dp]
inline size_t fid_dist_bytes(int D) { const size_t p = fid_pad(D); return FID_HDR + fid_al(p * 8) * 2 + fid_al(p * p * 8) * 4; }

__device__ __forceinline__ void dmma_16x8x4(double (&d)[4], double a0, double a1, double b0) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a0), "d"(a1), "d"(b0));
}

// fixed-order sum over a 256-thread block; the result is returned to every thread
__device__ __forceinline__ double fid_block_sum(double v, double* red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0;
    for (int w = 0; w < 8; ++w) t += red[w];
    return t;
}

// ---------------------------------------------------------------- statistics
// c (first batch: *init == 0) and s += sum_r (x[r] - c), per column; block (32 columns, 8 row groups), the groups combined in order
__global__ void __launch_bounds__(256) k_fid_colsum(const float* __restrict__ x, long long ld, int n, int D, const int* init,
                                                    double* c, double* s) {
    pdl_entry();
    __shared__ double part[8][32];
    const int j = blockIdx.x * 32 + threadIdx.x, g = threadIdx.y;
    const int per = (n + 7) / 8, r0 = g * per, r1 = min(n, r0 + per);
    const bool first = *init == 0;
    if (first) {
        double a = 0;
        if (j < D) for (int r = r0; r < r1; ++r) a += (double)x[(long long)r * ld + j];
        part[g][threadIdx.x] = a;
        __syncthreads();
        if (g == 0 && j < D) {
            double t = 0;
            for (int q = 0; q < 8; ++q) t += part[q][threadIdx.x];
            c[j] = t / (double)n;
        }
        __syncthreads();
    }
    const double cj = j < D ? c[j] : 0.0;
    double a = 0;
    if (j < D) for (int r = r0; r < r1; ++r) a += (double)x[(long long)r * ld + j] - cj;
    part[g][threadIdx.x] = a;
    __syncthreads();
    if (g == 0 && j < D) {
        double t = 0;
        for (int q = 0; q < 8; ++q) t += part[q][threadIdx.x];
        s[j] += t;
    }
}

struct FidGemm {
    const void* X; const void* Y;                // C[i][j] (+)= sum_k X(k, i) Y(k, j); X, Y row-major [K][ld]
    long long ldx, ldy;
    const double* shift;                         // statistics: X = Y = features - shift[col]; else null
    int K, ncols;                                // rows; valid columns (the rest read as 0)
    double* C; int ldc;
    int tiles;                                   // tiles per side
    int lower, accumulate;                       // lower: only tiles ti >= tj (grid = T(T+1)/2)
    const int* status;                           // skip everything when *status != 0 (null: never)
    int* set_init;                               // statistics: *set_init = 1 (the state now has its shift)
};

template <typename T>
__device__ __forceinline__ void fid_load_chunk(const T* __restrict__ X, long long ld, const double* shift, int k0, int K, int col0,
                                               int ncols, double (&r)[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int e = threadIdx.x + 256 * q, kr = e >> 6, col = col0 + (e & 63);
        double v = 0;
        if (k0 + kr < K && col < ncols) {
            v = (double)X[(long long)(k0 + kr) * ld + col];
            if (shift) v -= shift[col];
        }
        r[q] = v;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) k_fid_gemm(FidGemm p) {
    pdl_entry();
    if (p.status && *p.status) return;
    __shared__ double xs[FID_KC][FID_SPAD], ys[FID_KC][FID_SPAD];
    int ti, tj;
    if (p.lower) {
        const int t = blockIdx.x;
        ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
        while (ti * (ti + 1) / 2 > t) --ti;
        while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
        tj = t - ti * (ti + 1) / 2;
    } else {
        ti = blockIdx.x / p.tiles; tj = blockIdx.x % p.tiles;
    }
    if (p.set_init && blockIdx.x == 0 && threadIdx.x == 0) *p.set_init = 1;
    const T* X = static_cast<const T*>(p.X);
    const T* Y = static_cast<const T*>(p.Y);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, gid = lane >> 2, tig = lane & 3;
    const int wm = w & 3, wn = w >> 2;
    double acc[4][4] = {};
    double rx[4], ry[4];
    fid_load_chunk<T>(X, p.ldx, p.shift, 0, p.K, ti * FID_TILE, p.ncols, rx);
    fid_load_chunk<T>(Y, p.ldy, p.shift, 0, p.K, tj * FID_TILE, p.ncols, ry);
    for (int k0 = 0; k0 < p.K; k0 += FID_KC) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int e = threadIdx.x + 256 * q;
            xs[e >> 6][e & 63] = rx[q];
            ys[e >> 6][e & 63] = ry[q];
        }
        __syncthreads();
        if (k0 + FID_KC < p.K) {
            fid_load_chunk<T>(X, p.ldx, p.shift, k0 + FID_KC, p.K, ti * FID_TILE, p.ncols, rx);
            fid_load_chunk<T>(Y, p.ldy, p.shift, k0 + FID_KC, p.K, tj * FID_TILE, p.ncols, ry);
        }
#pragma unroll
        for (int kk = 0; kk < FID_KC; kk += 4) {
            const double a0 = xs[kk + tig][wm * 16 + gid], a1 = xs[kk + tig][wm * 16 + gid + 8];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) dmma_16x8x4(acc[nt], a0, a1, ys[kk + tig][wn * 32 + nt * 8 + gid]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = ti * FID_TILE + wm * 16 + gid + 8 * h, j = tj * FID_TILE + wn * 32 + nt * 8 + tig * 2;
            double* o = p.C + (long long)i * p.ldc + j;
            if (p.accumulate) { o[0] += acc[nt][2 * h]; o[1] += acc[nt][2 * h + 1]; }
            else { o[0] = acc[nt][2 * h]; o[1] = acc[nt][2 * h + 1]; }
        }
    }
}

// mean[i] = c[i] + s[i] / n;  cov[i][j] = (Cm[i][j] - s[i] s[j] / n) / (n - ddof), Cm read from its lower tile
__global__ void k_fid_finalize(const double* __restrict__ c, const double* __restrict__ s, const double* __restrict__ Cm, int Dp, int D,
                               double n, double denom, double* mean, double* cov) {
    pdl_entry();
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)D * D) return;
    const int i = (int)(e / D), j = (int)(e % D);
    const bool lo = i / FID_TILE >= j / FID_TILE;
    const double cm = lo ? Cm[(long long)i * Dp + j] : Cm[(long long)j * Dp + i];
    cov[e] = (cm - s[i] * s[j] / n) / denom;
    if (j == 0) mean[i] = c[i] + s[i] / n;
}

// ---------------------------------------------------------------- distance
__device__ __forceinline__ void fid_flag(int* status, int code) { atomicCAS(status, 0, code); }

// W[i][j] = (A[i][j] + A[j][i]) / 2 for i, j < D, 0 in the padding (Dp x Dp); V = I when given.  Non-finite A sets FID_NONFINITE.
__global__ void k_fid_sym(const double* __restrict__ A, long long lda, int D, int Dp, double* W, double* V, int* status) {
    pdl_entry();
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)Dp * Dp) return;
    const int i = (int)(e / Dp), j = (int)(e % Dp);
    double v = 0;
    if (i < D && j < D) {
        const double a = A[(long long)i * lda + j], b = A[(long long)j * lda + i];
        if (!isfinite(a)) fid_flag(status, FID_NONFINITE);
        v = 0.5 * (a + b);
    }
    W[e] = v;
    if (V) V[e] = i == j ? 1.0 : 0.0;
}

struct FidJacobi {
    double* W; double* V;                        // rows of A V and of V, pitch Dp
    int n, len, Dp;                              // n: players (D rounded up to even); len: elements per row touched
    double tol;
    int* counters;                               // [3] rotations of sweeps s % 3
    int* sweeps;
    int* status; int cap_code;
};

__device__ __forceinline__ void fid_pair(int r, int k, int n, int& a, int& b) {
    if (k == 0) { a = n - 1; b = r; }
    else { a = (r + k) % (n - 1); b = (r - k + (n - 1)) % (n - 1); }
}

// One-sided Jacobi, all sweeps in one cooperative launch.  No programmatic trigger: the next kernel starts after it completes.
__global__ void __launch_bounds__(256) k_fid_jacobi(FidJacobi p) {
    pdl_wait();
    cooperative_groups::grid_group grid = cooperative_groups::this_grid();
    if (*(volatile int*)p.status) return;
    __shared__ double red[3][8];
    __shared__ double cs[2];
    const int half = p.n / 2, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int sweep = 0;
    bool converged = false;
    for (; sweep < FID_MAX_SWEEPS && !converged; ++sweep) {
        if (blockIdx.x == 0 && threadIdx.x == 0) p.counters[(sweep + 1) % 3] = 0;
        for (int r = 0; r < p.n - 1; ++r) {
            for (int k = blockIdx.x; k < half; k += gridDim.x) {
                int a, b;
                fid_pair(r, k, p.n, a, b);
                double2* wa = reinterpret_cast<double2*>(p.W + (long long)a * p.Dp);
                double2* wb = reinterpret_cast<double2*>(p.W + (long long)b * p.Dp);
                double al = 0, be = 0, ga = 0;
                for (int e = threadIdx.x; e < p.len / 2; e += 256) {
                    const double2 x = wa[e], y = wb[e];
                    al = fma(x.x, x.x, fma(x.y, x.y, al));
                    be = fma(y.x, y.x, fma(y.y, y.y, be));
                    ga = fma(x.x, y.x, fma(x.y, y.y, ga));
                }
                for (int o = 16; o; o >>= 1) {
                    al += __shfl_xor_sync(0xffffffffu, al, o);
                    be += __shfl_xor_sync(0xffffffffu, be, o);
                    ga += __shfl_xor_sync(0xffffffffu, ga, o);
                }
                if (lane == 0) { red[0][w] = al; red[1][w] = be; red[2][w] = ga; }
                __syncthreads();
                if (threadIdx.x == 0) {
                    double A = 0, B = 0, G = 0;
                    for (int q = 0; q < 8; ++q) { A += red[0][q]; B += red[1][q]; G += red[2][q]; }
                    double c = 1, s = 0;
                    if (fabs(G) > p.tol * sqrt(A) * sqrt(B)) {
                        const double zeta = (B - A) / (2 * G);
                        const double t = fabs(zeta) > 1e150 ? 0.5 / zeta : copysign(1.0, zeta) / (fabs(zeta) + sqrt(1 + zeta * zeta));
                        c = 1 / sqrt(1 + t * t);
                        s = c * t;
                        atomicAdd(&p.counters[sweep % 3], 1);
                    }
                    cs[0] = c; cs[1] = s;
                }
                __syncthreads();
                const double c = cs[0], s = cs[1];
                if (s != 0) {
                    double2* va = reinterpret_cast<double2*>(p.V + (long long)a * p.Dp);
                    double2* vb = reinterpret_cast<double2*>(p.V + (long long)b * p.Dp);
                    for (int e = threadIdx.x; e < p.len / 2; e += 256) {
                        const double2 x = wa[e], y = wb[e], u = va[e], v = vb[e];
                        wa[e] = make_double2(c * x.x - s * y.x, c * x.y - s * y.y);
                        wb[e] = make_double2(s * x.x + c * y.x, s * x.y + c * y.y);
                        va[e] = make_double2(c * u.x - s * v.x, c * u.y - s * v.y);
                        vb[e] = make_double2(s * u.x + c * v.x, s * u.y + c * v.y);
                    }
                }
                __syncthreads();
            }
            grid.sync();
        }
        converged = *(volatile int*)&p.counters[sweep % 3] == 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *p.sweeps = sweep;
        if (!converged) fid_flag(p.status, p.cap_code);
    }
}

// lam[i] = sign(v_i . w_i) ||w_i||, one warp per row
__global__ void k_fid_eig(const double* __restrict__ W, const double* __restrict__ V, int D, int Dp, double* lam, const int* status) {
    pdl_entry();
    if (*status) return;
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= D) return;
    double nn = 0, dv = 0;
    for (int e = lane; e < D; e += 32) {
        const double x = W[(long long)i * Dp + e];
        nn = fma(x, x, nn);
        dv = fma(x, V[(long long)i * Dp + e], dv);
    }
    for (int o = 16; o; o >>= 1) { nn += __shfl_xor_sync(0xffffffffu, nn, o); dv += __shfl_xor_sync(0xffffffffu, dv, o); }
    if (lane == 0) lam[i] = dv < 0 ? -sqrt(nn) : sqrt(nn);
}

// ratio = lam_min / lam_max (0 when lam_max <= 0); below -FID_NEG_TOL flags code.  One block.
__global__ void __launch_bounds__(256) k_fid_eigcheck(const double* __restrict__ lam, int D, double* ratio_out, int* status, int code) {
    pdl_entry();
    if (*status) return;
    __shared__ double mx[256], mn[256];
    double a = -INFINITY, b = INFINITY;
    for (int i = threadIdx.x; i < D; i += 256) { a = fmax(a, lam[i]); b = fmin(b, lam[i]); }
    mx[threadIdx.x] = a; mn[threadIdx.x] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int q = 1; q < 256; ++q) { a = fmax(a, mx[q]); b = fmin(b, mn[q]); }
        const double r = a > 0 ? fmin(b, 0.0) / a : 0.0;
        *ratio_out = r;
        if (r < -FID_NEG_TOL) fid_flag(status, code);
    }
}

// L[k][i] = V[i][k] sqrt(max(lam_i, 0)) (i < D; 0 beyond), through a 32 x 32 shared tile
__global__ void k_fid_make_l(const double* __restrict__ V, const double* __restrict__ lam, int D, int Dp, double* L, const int* status) {
    pdl_entry();
    if (*status) return;
    __shared__ double t[32][33];
    const int i0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    for (int y = threadIdx.y; y < 32; y += 8) {
        const int i = i0 + y, k = k0 + threadIdx.x;
        t[y][threadIdx.x] = i < D ? V[(long long)i * Dp + k] * sqrt(fmax(lam[i], 0.0)) : 0.0;
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) L[(long long)(k0 + y) * Dp + i0 + threadIdx.x] = t[threadIdx.x][y];
}

// out = {fd, status, sweeps(S1), sweeps(M), lam_min/lam_max (S1), nu_min/nu_max (M), tr sqrt(S1 S2), 0}.  One block, fixed order.
__global__ void __launch_bounds__(256) k_fid_final(const double* __restrict__ mu1, const double* __restrict__ mu2, const double* __restrict__ S1,
                                                   const double* __restrict__ S2, const double* __restrict__ nu, int D, int* status,
                                                   const int* sweeps, double* out) {
    pdl_entry();
    __shared__ double red[8];
    double dd = 0, tr = 0, sq = 0;
    bool bad = false;
    for (int i = threadIdx.x; i < D; i += 256) {
        const double d = mu1[i] - mu2[i];
        bad |= !isfinite(d);
        dd = fma(d, d, dd);
        tr += S1[(long long)i * D + i] + S2[(long long)i * D + i];
    }
    if (bad) fid_flag(status, FID_NONFINITE);
    __syncthreads();
    const int st = *(volatile int*)status;
    if (st == 0)
        for (int i = threadIdx.x; i < D; i += 256) sq += sqrt(fmax(nu[i], 0.0));
    dd = fid_block_sum(dd, red);
    tr = fid_block_sum(tr, red);
    sq = fid_block_sum(sq, red);
    if (threadIdx.x == 0) {
        out[0] = st ? NAN : dd + tr - 2 * sq;
        out[1] = st;
        out[2] = sweeps[0]; out[3] = sweeps[1];
        out[6] = st ? NAN : sq;
        out[7] = 0;
    }
}

// ---------------------------------------------------------------- host
inline cudaError_t fid_stats_launch(void* state, int D, const float* feats, long long n, long long ld, cudaStream_t st) {
    const int Dp = fid_pad(D), T = Dp / FID_TILE;
    char* b = static_cast<char*>(state);
    int* init = reinterpret_cast<int*>(b);
    double* c = reinterpret_cast<double*>(b + FID_HDR);
    double* s = reinterpret_cast<double*>(b + FID_HDR + fid_al((size_t)Dp * 8));
    double* Cm = reinterpret_cast<double*>(b + FID_HDR + 2 * fid_al((size_t)Dp * 8));
    cudaError_t e = launch_k(k_fid_colsum, dim3((D + 31) / 32), dim3(32, 8), 0, st, feats, ld, (int)n, D, (const int*)init, c, s);
    if (e != cudaSuccess) return e;
    FidGemm g{feats, feats, ld, ld, c, (int)n, D, Cm, Dp, T, 1, 1, nullptr, init};
    return launch_k(k_fid_gemm<float>, dim3(T * (T + 1) / 2), dim3(256), 0, st, g);
}

inline cudaError_t fid_finalize_launch(const void* state, int D, long long n, int ddof, double* mean, double* cov, cudaStream_t st) {
    const int Dp = fid_pad(D);
    const char* b = static_cast<const char*>(state);
    const double* c = reinterpret_cast<const double*>(b + FID_HDR);
    const double* s = reinterpret_cast<const double*>(b + FID_HDR + fid_al((size_t)Dp * 8));
    const double* Cm = reinterpret_cast<const double*>(b + FID_HDR + 2 * fid_al((size_t)Dp * 8));
    const long long tot = (long long)D * D;
    return launch_k(k_fid_finalize, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, c, s, Cm, Dp, D, (double)n,
                    (double)(n - ddof), mean, cov);
}

inline cudaError_t fid_jacobi_launch(const FidJacobi& j, cudaStream_t st) {
    int dev = 0, sms = 0, per = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_fid_jacobi, 256, 0);
    if (e != cudaSuccess) return e;
    const int grid = std::max(1, std::min(j.n / 2, per * sms));
    cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256); cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k_fid_jacobi, j);
}

inline cudaError_t fid_distance_launch(const double* mu1, const double* S1, const double* mu2, const double* S2, int D, double* out,
                                       void* scratch, cudaStream_t st) {
    const int Dp = fid_pad(D), T = Dp / FID_TILE;
    const size_t vec = fid_al((size_t)Dp * 8), mat = fid_al((size_t)Dp * Dp * 8);
    char* b = static_cast<char*>(scratch);
    int* status = reinterpret_cast<int*>(b);
    int* counters = status + 1;                  // [2][3]: one set per eigen-solve
    int* sweeps = status + 7;
    double* lam = reinterpret_cast<double*>(b + FID_HDR);
    double* nu = reinterpret_cast<double*>(b + FID_HDR + vec);
    double* W = reinterpret_cast<double*>(b + FID_HDR + 2 * vec);
    double* V = reinterpret_cast<double*>(b + FID_HDR + 2 * vec + mat);
    double* S2p = reinterpret_cast<double*>(b + FID_HDR + 2 * vec + 2 * mat);
    double* L = reinterpret_cast<double*>(b + FID_HDR + 2 * vec + 3 * mat);
    const int n = (D + 1) & ~1;
    const double tol = (double)D * 0x1p-53;
    const unsigned eb = (unsigned)(((long long)Dp * Dp + 255) / 256);
    cudaError_t e;
#define FID_TRY(x) if ((e = (x)) != cudaSuccess) return e
    FID_TRY(cudaMemsetAsync(status, 0, 9 * sizeof(int), st));
    FID_TRY(launch_k(k_fid_sym, dim3(eb), dim3(256), 0, st, S1, (long long)D, D, Dp, W, V, status));
    FID_TRY(launch_k(k_fid_sym, dim3(eb), dim3(256), 0, st, S2, (long long)D, D, Dp, S2p, (double*)nullptr, status));
    FID_TRY(fid_jacobi_launch(FidJacobi{W, V, n, n, Dp, tol, counters, sweeps, status, FID_NO_CONV_1}, st));
    FID_TRY(launch_k(k_fid_eig, dim3((D + 7) / 8), dim3(256), 0, st, (const double*)W, (const double*)V, D, Dp, lam, (const int*)status));
    FID_TRY(launch_k(k_fid_eigcheck, dim3(1), dim3(256), 0, st, (const double*)lam, D, out + 4, status, (int)FID_NOT_PSD_1));
    FID_TRY(launch_k(k_fid_make_l, dim3(Dp / 32, Dp / 32), dim3(32, 8), 0, st, (const double*)V, (const double*)lam, D, Dp, L, (const int*)status));
    // P = S2^T L into W (S2 is symmetric), then M = L^T P into V
    FidGemm g1{S2p, L, Dp, Dp, nullptr, Dp, Dp, W, Dp, T, 0, 0, status, nullptr};
    FID_TRY(launch_k(k_fid_gemm<double>, dim3(T * T), dim3(256), 0, st, g1));
    FidGemm g2{L, W, Dp, Dp, nullptr, Dp, Dp, V, Dp, T, 0, 0, status, nullptr};
    FID_TRY(launch_k(k_fid_gemm<double>, dim3(T * T), dim3(256), 0, st, g2));
    FID_TRY(launch_k(k_fid_sym, dim3(eb), dim3(256), 0, st, (const double*)V, (long long)Dp, D, Dp, W, L, status));
    FID_TRY(fid_jacobi_launch(FidJacobi{W, L, n, n, Dp, tol, counters + 3, sweeps + 1, status, FID_NO_CONV_M}, st));
    FID_TRY(launch_k(k_fid_eig, dim3((D + 7) / 8), dim3(256), 0, st, (const double*)W, (const double*)L, D, Dp, nu, (const int*)status));
    FID_TRY(launch_k(k_fid_eigcheck, dim3(1), dim3(256), 0, st, (const double*)nu, D, out + 5, status, (int)FID_NOT_PSD_M));
    FID_TRY(launch_k(k_fid_final, dim3(1), dim3(256), 0, st, mu1, mu2, S1, S2, (const double*)nu, D, status, (const int*)sweeps, out));
#undef FID_TRY
    return cudaSuccess;
}

}  // namespace ddpm
