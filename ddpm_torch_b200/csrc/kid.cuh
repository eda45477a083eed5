// Kernel Inception Distance (Bińkowski et al., 2018): the unbiased polynomial-kernel MMD^2 between two feature sets, averaged over
// subsets, as torch-fidelity and clean-fid compute it.
//
// With k(x, y) = (gamma x . y + c0)^degree and, for subset s, rows ix (of X) and iy (of Y), m each:
//   mmd2_s = (sum_{i != j} k(x_i, x_j) + sum_{i != j} k(y_i, y_j)) / (m (m - 1)) - 2 sum_{i, j} k(x_i, y_j) / m^2.
// The three sums are of ~m^2 terms of order 1 whose difference is often 1e-3 .. 1e-4 of them, so the Gram entries and every sum
// are fp64: fp32 x fp32 products are exact in fp64, and the DMMA (mma.sync m16n8k4 f64) tensor core accumulates them in fp64.
//
//   k_kid_tiles   one CTA per (subset, 64 x 64 tile): the upper triangle (diagonal tiles included) of XX, that of YY, and every
//                 tile of XY.  It gathers its 2 x 64 rows by index from the fp32 features, converts them to fp64 in shared memory
//                 chunk by chunk along d, accumulates the Gram tile with DMMA, and in the epilogue applies the kernel (repeated
//                 multiplication), drops i == j in the XX / YY diagonal tiles and the padding past m, and reduces the tile in a
//                 fixed order (fid_block_sum) to one fp64 partial; an off-diagonal XX / YY tile counts twice (k is symmetric).
//                 Each partial has its own slot: no atomics.
//   k_kid_finish  one CTA: per subset the XX, YY and XY partials summed in tile order, then mmd2_s, the mean and the population
//                 std over subsets; the status is 1 when any subset's sum is not finite (a non-finite feature in a drawn row, or a
//                 kernel value that overflows).
// Every sum has a fixed order that depends on (S, m) only, so the result is bit-identical from run to run and depends on the
// drawn feature rows alone, not on how the features were batched.
#pragma once
#include "fid.cuh"

namespace ddpm {

constexpr int KID_TILE = 64;                    // Gram tile
constexpr int KID_KC = 32;                      // feature columns per shared-memory chunk (one 128-byte fp32 row segment)
constexpr int KID_SPAD = KID_KC + 4;            // row pitch (doubles) of the shared tiles: conflict-free fragment loads
constexpr int KID_MAX_DEGREE = 8;

// ddpm_kid's status (out[S + 2])
enum KidStatus { KID_OK = 0, KID_NONFINITE = 1 };

inline int kid_tiles(int m) { return (m + KID_TILE - 1) / KID_TILE; }
// partials per subset: XX upper triangle | YY upper triangle | XY
inline long long kid_blocks(int m) { const long long T = kid_tiles(m); return T * (T + 1) + T * T; }
// scratch: indices i32[S][2][m] | partials f64[S][kid_blocks(m)]
inline size_t kid_idx_bytes(int S, int m) { return fid_al((size_t)S * 2 * m * 4); }
inline size_t kid_bytes(int S, int m) { return kid_idx_bytes(S, m) + fid_al((size_t)S * kid_blocks(m) * 8); }

struct KidArgs {
    const float* x; const float* y;             // fp32 feature rows, pitches ldx / ldy
    long long ldx, ldy;
    const int* idx;                             // [S][2][m]: ix then iy, in range and distinct (checked on the host)
    int d, m, T, nb, degree;                    // T tiles per side, nb = kid_blocks(m)
    double gamma, coef0;
    double* partial;                            // [S][nb]
};

// The chunk [k0, k0 + KID_KC) of 64 gathered rows into registers: thread e = threadIdx.x + 256 q takes row e / 32, column e % 32,
// so a warp reads one row's 128 contiguous bytes.  Rows past m and columns past d read as 0.
__device__ __forceinline__ void kid_load_chunk(const float* __restrict__ X, const long long* off, int k0, int d, float (&r)[8]) {
    const int c = k0 + (threadIdx.x & 31);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const long long o = off[(threadIdx.x >> 5) + 8 * q];
        r[q] = o >= 0 && c < d ? X[o + c] : 0.f;
    }
}

__device__ __forceinline__ void kid_store_chunk(double (*s)[KID_SPAD], const float (&r)[8]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) s[(threadIdx.x >> 5) + 8 * q][threadIdx.x & 31] = (double)r[q];
}

__global__ void __launch_bounds__(256) k_kid_tiles(KidArgs p) {
    pdl_entry();
    __shared__ double xs[KID_TILE][KID_SPAD], ys[KID_TILE][KID_SPAD];
    __shared__ long long offa[KID_TILE], offb[KID_TILE];
    __shared__ double red[8];
    const int s = blockIdx.x / p.nb, b = blockIdx.x - s * p.nb, tu = p.T * (p.T + 1) / 2;
    int kind, ti, tj;                           // kind 0: XX, 1: YY, 2: XY
    if (b < 2 * tu) {
        kind = b >= tu;
        fid_tri_tile(b - kind * tu, tj, ti);    // ti <= tj
    } else {
        kind = 2;
        ti = (b - 2 * tu) / p.T; tj = (b - 2 * tu) % p.T;
    }
    const float* A = kind == 1 ? p.y : p.x;
    const float* B = kind == 0 ? p.x : p.y;
    const long long lda = kind == 1 ? p.ldy : p.ldx, ldb = kind == 0 ? p.ldx : p.ldy;
    const int* ia = p.idx + (long long)s * 2 * p.m + (kind == 1 ? p.m : 0);
    const int* ib = p.idx + (long long)s * 2 * p.m + (kind == 0 ? 0 : p.m);
    if (threadIdx.x < 2 * KID_TILE) {
        const int r = threadIdx.x & (KID_TILE - 1), hi = threadIdx.x >= KID_TILE;
        const int i = (hi ? tj : ti) * KID_TILE + r;
        (hi ? offb : offa)[r] = i < p.m ? (long long)(hi ? ib : ia)[i] * (hi ? ldb : lda) : -1;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, gid = lane >> 2, tig = lane & 3;
    const int wm = w & 3, wn = w >> 2;
    double acc[4][4] = {};
    float ra[8], rb[8];
    kid_load_chunk(A, offa, 0, p.d, ra);
    kid_load_chunk(B, offb, 0, p.d, rb);
    for (int k0 = 0; k0 < p.d; k0 += KID_KC) {
        kid_store_chunk(xs, ra);
        kid_store_chunk(ys, rb);
        __syncthreads();
        if (k0 + KID_KC < p.d) {
            kid_load_chunk(A, offa, k0 + KID_KC, p.d, ra);
            kid_load_chunk(B, offb, k0 + KID_KC, p.d, rb);
        }
#pragma unroll
        for (int kk = 0; kk < KID_KC; kk += 4) {
            const double a0 = xs[wm * 16 + gid][kk + tig], a1 = xs[wm * 16 + gid + 8][kk + tig];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) dmma_16x8x4(acc[nt], a0, a1, ys[wn * 32 + nt * 8 + gid][kk + tig]);
        }
        __syncthreads();
    }
    double sum = 0;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int i = ti * KID_TILE + wm * 16 + gid + 8 * (e >> 1), j = tj * KID_TILE + wn * 32 + nt * 8 + tig * 2 + (e & 1);
            if (i < p.m && j < p.m && (kind == 2 || i != j)) {
                const double base = p.gamma * acc[nt][e] + p.coef0;
                double v = base;
                for (int q = 1; q < p.degree; ++q) v *= base;
                sum += v;
            }
        }
    }
    sum = fid_block_sum(sum, red);
    if (threadIdx.x == 0) p.partial[blockIdx.x] = kind != 2 && ti != tj ? 2 * sum : sum;
}

// out[0..S) = mmd2_s, out[S] = mean, out[S + 1] = population std, out[S + 2] = status (mean and std NaN when it is not 0)
__global__ void __launch_bounds__(256) k_kid_finish(const double* __restrict__ partial, int S, int m, int nb, int tu, double* out) {
    pdl_entry();
    __shared__ double red[8];
    const double dxx = (double)m * (double)(m - 1), dxy = (double)m * (double)m;
    double tot = 0, bad = 0;
    for (int s = threadIdx.x; s < S; s += 256) {
        const double* q = partial + (long long)s * nb;
        double xx = 0, yy = 0, xy = 0;
        for (int b = 0; b < tu; ++b) xx += q[b];
        for (int b = tu; b < 2 * tu; ++b) yy += q[b];
        for (int b = 2 * tu; b < nb; ++b) xy += q[b];
        if (!isfinite(xx) || !isfinite(yy) || !isfinite(xy)) bad = 1;
        const double v = (xx + yy) / dxx - 2 * xy / dxy;
        out[s] = v;
        tot += v;
    }
    const double mean = fid_block_sum(tot, red) / S;
    double sq = 0;
    for (int s = threadIdx.x; s < S; s += 256) { const double e = out[s] - mean; sq += e * e; }
    sq = fid_block_sum(sq, red);
    bad = fid_block_sum(bad, red);
    if (threadIdx.x == 0) {
        out[S] = bad ? (double)NAN : mean;
        out[S + 1] = bad ? (double)NAN : sqrt(sq / S);
        out[S + 2] = bad ? (double)KID_NONFINITE : (double)KID_OK;
    }
}

// idx_host [S][2][m] (checked by the caller) is copied into the scratch (kid_bytes(S, m)) on st; then the two kernels
inline cudaError_t kid_launch(const float* x, long long ldx, const float* y, long long ldy, int d, const int* idx_host, int S, int m,
                              int degree, double gamma, double coef0, double* out, void* scratch, cudaStream_t st) {
    int* idx = static_cast<int*>(scratch);
    double* partial = reinterpret_cast<double*>(static_cast<char*>(scratch) + kid_idx_bytes(S, m));
    cudaError_t e = cudaMemcpyAsync(idx, idx_host, (size_t)S * 2 * m * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    const int T = kid_tiles(m), nb = (int)kid_blocks(m);
    const KidArgs a{x, y, ldx, ldy, idx, d, m, T, nb, degree, gamma, coef0, partial};
    e = launch_k(k_kid_tiles, dim3((unsigned)((long long)S * nb)), dim3(256), 0, st, a);
    if (e != cudaSuccess) return e;
    return launch_k(k_kid_finish, dim3(1), dim3(256), 0, st, (const double*)partial, S, m, nb, T * (T + 1) / 2, out);
}

}  // namespace ddpm
