// Inception Score (Salimans et al., 2016; the TensorFlow improved-gan/inception_score.py that papers report): the 1008-way logits
// of the FID Inception's pool3 features and the per-split exp(KL(p(y|x) || p(y))).
//
// Logits.  logits = pool3 . W^T with W the checkpoint's fc.weight [1008][2048] and no bias (the TF graph multiplies by the
// softmax/logits/MatMul weight alone).  A single TF32 product would leave a logit of ~10 off by ~5e-3, which moves p by ~0.5 %, so
// the GEMM is 3xTF32 through the Inception convolution kernel's body (inc_conv_tf32_body, no bias, no ReLU): a 1 x 1 convolution
// over N one-pixel images with K = 3 x 2048, the features split by k_is_split into [f_hi | f_lo | f_hi] and the weights packed by
// k_is_pack as [w_hi | w_hi | w_lo], so each output is f_hi w_hi + f_lo w_hi + f_hi w_lo summed in fp32.  No split-K, no atomics:
// a logit depends on its image's features only.
//
// Score, in fp64 on the fp32 logits z [N][C] (C = 1008 for the network), with every reduction in a fixed order:
//   k_is_rows   per row x, in one pass over d = z - max z: lse_x = max z + log s with s = sum exp(d), and the row term
//               t_x = sum_y p_xy (z_xy - lse_x) = (sum exp(d) d) / s - log s; log p is z - lse, never the log of a rounded
//               softmax, so a saturated row stays finite.
//               A non-finite logit sets the status.
//   k_is_cols   per part i (rows [i N / splits, (i + 1) N / splits)), row chunk and column: the chunk's sum of p_xy, rows in order.
//   k_is_final  per part: pbar_y = (sum of its chunks, in order) / n_i and KL_i = (sum_x t_x) / n_i - sum_y pbar_y log pbar_y
//               (0 log 0 = 0), out[i] = exp(KL_i); out[splits] = the status.
// The chunking depends on (N, splits) only, so the score of given logits is bit-identical from call to call, and (the logits being
// per-image) however the images were batched through the network.
#pragma once
#include "inception.cuh"
#include "fid.cuh"

namespace ddpm {

constexpr int IS_FEAT = 2048;                  // pool3 features
constexpr int IS_CLASSES = 1008;               // the network's fc outputs
constexpr int IS_K = 3 * IS_FEAT;              // the split GEMM's K
constexpr int IS_BN = 128;                     // logits GEMM tile width (1008 -> 8 tiles)
constexpr int IS_MAX_CHUNKS = 32;              // row chunks per part of the column sums
constexpr int IS_CHUNK_ROWS = 128;             // fewest rows a chunk is given
constexpr int IS_COUT_PAD = (IS_CLASSES + INC_COUT_PAD - 1) / INC_COUT_PAD * INC_COUT_PAD;
constexpr size_t IS_HDR = 256;

// ddpm_is_score's status (out[splits])
enum IsStatus { IS_OK = 0, IS_NONFINITE = 1 };

inline size_t is_packed_bytes() { return (size_t)IS_COUT_PAD * IS_K * 4; }
inline size_t is_logits_ws_bytes(int N) { return inc_al256((size_t)N * IS_K * 4); }
inline int is_chunks(int N, int splits) {
    const int c = N / splits / IS_CHUNK_ROWS;
    return c < 1 ? 1 : c > IS_MAX_CHUNKS ? IS_MAX_CHUNKS : c;
}
__host__ __device__ inline int is_col_blocks(int C) { return (C + 255) / 256; }
// scratch: header (status) | lse f64[N] | t f64[N] | partial column sums f64[splits][chunks][C]
inline size_t is_score_bytes(int N, int C, int splits) {
    return IS_HDR + 2 * fid_al((size_t)N * 8) + fid_al((size_t)splits * is_chunks(N, splits) * C * 8);
}

// ------------------------------------------------------------------------------------------------ logits
// wp [1024][IS_K]: row co < 1008 is [w_hi | w_hi | w_lo] of fc.weight[co] with w_hi = tf32(w), w_lo = tf32(w - w_hi); rows past 1008 zero
__global__ void k_is_pack(const float* __restrict__ w, float* __restrict__ wp) {
    pdl_entry();
    const long long total = (long long)IS_COUT_PAD * IS_K;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i / IS_K), k = (int)(i - (long long)co * IS_K), part = k / IS_FEAT, c = k - part * IS_FEAT;
        float v = 0.f;
        if (co < IS_CLASSES) {
            const float f = w[(long long)co * IS_FEAT + c], hi = __uint_as_float(tf32_rna(f));
            v = part < 2 ? hi : __uint_as_float(tf32_rna(f - hi));
        }
        wp[i] = v;
    }
}

// features [N] rows of pitch ld -> [N][IS_K] = [f_hi | f_lo | f_hi], f_hi = tf32(f), f_lo = f - f_hi (exact)
__global__ void k_is_split(const float* __restrict__ f, long long ld, int N, float* __restrict__ out) {
    pdl_entry();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)N * IS_FEAT; i += (long long)gridDim.x * blockDim.x) {
        const long long n = i / IS_FEAT;
        const int c = (int)(i - n * IS_FEAT);
        const float v = f[n * ld + c], hi = __uint_as_float(tf32_rna(v));
        float* o = out + n * IS_K + c;
        o[0] = hi; o[IS_FEAT] = v - hi; o[2 * IS_FEAT] = hi;
    }
}

__global__ void __launch_bounds__(INC_THREADS, 1) is_logits_tf32_kernel(const IncConvArgs a) { inc_conv_tf32_body<IS_BN, false>(a); }

inline cudaError_t is_pack_launch(const float* w, float* wp, cudaStream_t st) {
    return launch_k(k_is_pack, dim3(inc_grid((long long)IS_COUT_PAD * IS_K)), dim3(256), 0, st, w, wp);
}

// logits [N][IS_CLASSES] (row pitch IS_CLASSES) of features [N] (row pitch ld); ws: is_logits_ws_bytes(N)
inline cudaError_t is_logits_launch(const float* wp, const float* feats, long long ld, int N, float* logits, void* ws, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        const cudaError_t e = cudaFuncSetAttribute(is_logits_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, inc_smem_bytes<IS_BN>());
        if (e != cudaSuccess) return e;
        attr = true;
    }
    float* split = static_cast<float*>(ws);
    cudaError_t e = launch_k(k_is_split, dim3(inc_grid((long long)N * IS_FEAT)), dim3(256), 0, st, feats, ld, N, split);
    if (e != cudaSuccess) return e;
    IncConvArgs a;
    a.x = split; a.H = 1; a.W = 1; a.Cin4 = IS_K;
    a.Ho = 1; a.Wo = 1; a.kw = 1; a.stride = 1; a.ph = 0; a.pw = 0;
    a.K = IS_K; a.KT = IS_K / INC_BK;
    a.w = wp; a.bias = nullptr; a.out = logits; a.Cout = IS_CLASSES; a.c_off = 0; a.C_total = IS_CLASSES;
    a.M = N; a.n_tiles = (IS_CLASSES + IS_BN - 1) / IS_BN;
    const long long grid = (long long)((N + INC_BM - 1) / INC_BM) * a.n_tiles;
    return launch_k(is_logits_tf32_kernel, dim3((unsigned)grid), dim3(INC_THREADS), inc_smem_bytes<IS_BN>(), st, a);
}

// ------------------------------------------------------------------------------------------------ score
// one warp per row; the lanes' column-order partial sums are combined by an xor butterfly (the same value on every lane)
__global__ void __launch_bounds__(256) k_is_rows(const float* __restrict__ z, long long ld, int N, int C, double* __restrict__ lse,
                                                 double* __restrict__ term, int* status) {
    pdl_entry();
    const int lane = threadIdx.x & 31;
    const long long x = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (x >= N) return;
    const float* r = z + x * ld;
    float m = -INFINITY;
    bool fin = true;
    for (int y = lane; y < C; y += 32) {
        const float v = r[y];
        fin &= isfinite(v);
        m = fmaxf(m, v);
    }
    if (!__all_sync(0xffffffffu, fin)) {
        if (lane == 0) { atomicCAS(status, 0, (int)IS_NONFINITE); lse[x] = 0.0; term[x] = 0.0; }
        return;
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // with d = z - max and s = sum e^d: lse = max + log s and t = sum (e^d / s)(d - log s) = (sum e^d d) / s - log s
    double s = 0.0, u = 0.0;
#pragma unroll 4
    for (int y = lane; y < C; y += 32) {
        const double d = (double)r[y] - (double)m, e = exp(d);
        s += e; u += e * d;
    }
    for (int o = 16; o; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); u += __shfl_xor_sync(0xffffffffu, u, o); }
    if (lane == 0) { const double ls = log(s); lse[x] = (double)m + ls; term[x] = u / s - ls; }
}

// block = (part, chunk, 256 columns); a thread sums p over its chunk's rows in order
__global__ void __launch_bounds__(256) k_is_cols(const float* __restrict__ z, long long ld, int N, int C, int splits, int chunks,
                                                 const double* __restrict__ lse, double* __restrict__ partial) {
    pdl_entry();
    const int cblocks = is_col_blocks(C);
    const int pc = blockIdx.x / cblocks, y = (blockIdx.x - pc * cblocks) * 256 + threadIdx.x;
    const int part = pc / chunks, ch = pc - part * chunks;
    if (y >= C) return;
    const long long b = (long long)part * N / splits, n = (long long)(part + 1) * N / splits - b;
    const long long r0 = b + n * ch / chunks, r1 = b + n * (ch + 1) / chunks;
    double s = 0.0;
    for (long long x = r0; x < r1; ++x) s += exp((double)z[x * ld + y] - lse[x]);
    partial[(long long)pc * C + y] = s;
}

// one 256-thread block per part
__global__ void __launch_bounds__(256) k_is_final(const double* __restrict__ term, const double* __restrict__ partial, int N, int C,
                                                  int splits, int chunks, const int* __restrict__ status, double* __restrict__ out) {
    pdl_entry();
    __shared__ double red[8];
    const int part = blockIdx.x;
    const long long b = (long long)part * N / splits, e = (long long)(part + 1) * N / splits;
    const double n = (double)(e - b);
    double ent = 0.0;
    for (int y = threadIdx.x; y < C; y += 256) {
        double s = 0.0;
        for (int c = 0; c < chunks; ++c) s += partial[((long long)part * chunks + c) * C + y];
        const double pb = s / n;
        if (pb > 0.0) ent += pb * log(pb);
    }
    ent = fid_block_sum(ent, red);
    double t = 0.0;
    for (long long x = b + threadIdx.x; x < e; x += 256) t += term[x];
    t = fid_block_sum(t, red);
    if (threadIdx.x == 0) {
        const int st = *status;
        out[part] = st ? (double)NAN : exp(t / n - ent);
        if (part == 0) out[splits] = (double)st;
    }
}

// out[0..splits) = IS_i, out[splits] = status; scratch: is_score_bytes(N, C, splits)
inline cudaError_t is_score_launch(const float* z, long long ld, int N, int C, int splits, double* out, void* scratch, cudaStream_t st) {
    const int chunks = is_chunks(N, splits);
    uint8_t* p = static_cast<uint8_t*>(scratch);
    int* status = reinterpret_cast<int*>(p);
    double* lse = reinterpret_cast<double*>(p + IS_HDR);
    double* term = reinterpret_cast<double*>(p + IS_HDR + fid_al((size_t)N * 8));
    double* partial = reinterpret_cast<double*>(p + IS_HDR + 2 * fid_al((size_t)N * 8));
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int), st);
    if (e == cudaSuccess) e = launch_k(k_is_rows, dim3((unsigned)((N + 7) / 8)), dim3(256), 0, st, z, ld, N, C, lse, term, status);
    if (e == cudaSuccess)
        e = launch_k(k_is_cols, dim3((unsigned)((long long)splits * chunks * is_col_blocks(C))), dim3(256), 0, st, z, ld, N, C, splits,
                     chunks, (const double*)lse, partial);
    if (e == cudaSuccess)
        e = launch_k(k_is_final, dim3((unsigned)splits), dim3(256), 0, st, (const double*)term, (const double*)partial, N, C, splits,
                     chunks, (const int*)status, out);
    return e;
}

}  // namespace ddpm
