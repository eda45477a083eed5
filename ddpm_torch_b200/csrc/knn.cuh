// k-nearest-neighbour radii and manifold coverage of the improved precision/recall metric (ddpm_torch/metrics/precision_recall.py).
// The reference materialises fp16 torch.cdist blocks and runs kthvalue / `<=`.any() on them on the host (:43-55, :156-164, :177-206);
// here one fp16 wgmma GEMM per pass feeds a selection epilogue and no distance ever leaves the chip.
//
// Numerics (the fp16 features exactly as stored):
//   na[i] = sum_d a[i,d]^2 in fp32 (k_knn_norms, fixed order);  d2[i,j] = max(0, (na[i] + nb[j]) - 2 <a_i, b_j>), the inner product
//   on fp16 wgmma with fp32 accumulation;  kth[i] = fp16_rn(sqrt_rn(kk-th smallest d2[i, .]));  row i is covered iff
//   exists j: fp16_rn(sqrt_rn(d2[i,j])) <= r[j].  fp16 o sqrt is monotone, so this is the reference's formula with exact distances
//   in place of fp16 cdist.  The density of density/coverage (Naeem et al., 2020) counts instead, with a strict comparison:
//   count[i] = #{j : fp16_rn(sqrt_rn(d2[i,j])) < r[j]}.  Values only, no atomics: two calls on the same inputs are bit-identical.
//
// Layout: the engine's warp-specialised persistent kernel.  Warpgroup 0 is the TMA producer, warpgroups 1-2 each own 64 rows of a
// 128-row tile; 64-wide fp16 K slabs with 128-byte swizzle flow through a 4-stage mbarrier pipeline.  A work item is one row tile x a
// contiguous range of 256-column tiles (a column split); the consumers keep per-row state (a register list of the kk smallest d2, a
// coverage flag or a count) across all column tiles of the range, merge it over the quad of lanes that share a row, and write one
// entry per (split, row) to scratch.  A small finalise kernel merges the splits.  Items run split-fastest, so CTAs that run together
// share their row tile and walk the same column tiles (both operands are then mostly served from L2).
#pragma once
#include <algorithm>
#include <cuda_fp16.h>
#include "gemm_host.cuh"
#include "wgmma.cuh"

namespace ddpm {

constexpr int KNN_MAX_K = 16;                    // kk = nhood_size + 1 <= 16: the register lists of the kth epilogue
constexpr int KNN_BN = 256;                      // columns per tile (m64n256k16 per consumer warpgroup)
constexpr int KNN_STAGES = 4;
constexpr int KNN_A_BYTES = 128 * 128;           // 128 rows x 64 fp16
constexpr int KNN_B_BYTES = KNN_BN * 128;
constexpr int KNN_STAGE_BYTES = KNN_A_BYTES + KNN_B_BYTES;
constexpr int KNN_SMEM = 1024 /*align slack*/ + KNN_STAGES * KNN_STAGE_BYTES + 3 * KNN_BN * 4 + 2 * KNN_STAGES * 8;
enum KnnMode { KNN_KTH = 0, KNN_COVER = 1, KNN_COUNT = 2 };

struct KnnParams {
    int n_rows, n_cols, kblocks;                 // kblocks = ceil(D / 64)
    int m_tiles, n_tiles, splits, per_split;     // item t: row tile t / splits, column tiles [s * per_split, ...) with s = t % splits
    int kk;                                      // kth: list length written per (split, row)
    const float* na; const float* nb;            // squared norms of the rows / columns
    const __half* radii;                         // cover, count: r[n_cols]
    float* part;                                 // kth: [splits][n_rows][kk]
    uint8_t* flags;                              // cover: [splits][n_rows]
    int* counts;                                 // count: [splits][n_rows]
};

__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// ascending list of the KNN_MAX_K smallest values seen: a branch-free insertion (compile-time indices keep it in registers)
__device__ __forceinline__ void knn_insert(float (&l)[KNN_MAX_K], float v) {
#pragma unroll
    for (int i = 0; i < KNN_MAX_K; ++i) { const float lo = fminf(l[i], v); v = fmaxf(l[i], v); l[i] = lo; }
}
__device__ __forceinline__ float knn_at(const float (&l)[KNN_MAX_K], int k) {
    float r = l[0];
#pragma unroll
    for (int i = 1; i < KNN_MAX_K; ++i) if (i == k) r = l[i];
    return r;
}
// the contract's coverage test of one distance: fp16_rn(sqrt_rn(d2)) <= r (compared as values, like the reference's fp16 `<=`)
__device__ __forceinline__ bool knn_le(float d2, float r) { return __half2float(__float2half_rn(__fsqrt_rn(d2))) <= r; }
// the density test of one distance: fp16_rn(sqrt_rn(d2)) < r (so a radius of 0, a negative radius or NaN contains nothing)
__device__ __forceinline__ bool knn_lt(float d2, float r) { return __half2float(__float2half_rn(__fsqrt_rn(d2))) < r; }
// a d2 above this bound can never pass knn_le(d2, r), nor therefore knn_lt: fp16_rn(sqrt(d2)) <= r needs sqrt(d2) below the next
// fp16 above r.
// (the 2^-10 margin covers the fp32 rounding of the square; -1 for a negative radius, which no distance can meet)
__device__ __forceinline__ float knn_cover_bound(__half r) {
    const float rf = __half2float(r);
    if (!(rf >= 0.f)) return -1.f;
    const unsigned short b = __half_as_ushort(r) & 0x7fff;
    if (b >= 0x7c00) return INFINITY;
    const float up = __half2float(__ushort_as_half((unsigned short)(b + 1)));
    return up * up * (1.f + 0x1p-10f);
}

// The pass shared by every mode: main loop, column vectors and the per-mode epilogue.  The __global__ wrappers below pass their
// __grid_constant__ parameters by reference, so the tensor maps are still read from parameter space.
template <int MODE>
__device__ __forceinline__ void knn_wgmma_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const KnnParams& p) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_nb = reinterpret_cast<float*>(smem + KNN_STAGES * KNN_STAGE_BYTES);   // [KNN_BN] nb of the current column tile
    float* s_thr = s_nb + KNN_BN;                                                   // cover, count: knn_cover_bound(r)
    float* s_rf = s_thr + KNN_BN;                                                   // cover, count: r as float
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_rf + KNN_BN);
    uint64_t* empty_bar = full_bar + KNN_STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int items = p.m_tiles * p.splits;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
        for (int s = 0; s < KNN_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], EPI_THREADS / 32); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();

    if (threadIdx.x < 128) {
        // ======================= TMA producer =======================
        reg_dealloc<PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            int stg = 0;
            for (int t = blockIdx.x; t < items; t += gridDim.x) {
                const int mt = t / p.splits, c0 = (t % p.splits) * p.per_split;
                const int c1 = min(p.n_tiles, c0 + p.per_split);
                for (int ct = c0; ct < c1; ++ct)
                    for (int kb = 0; kb < p.kblocks; ++kb, ++stg) {
                        const int st = stg % KNN_STAGES;
                        if (!mbar_wait(&empty_bar[st], ((stg / KNN_STAGES) & 1) ^ 1, 11)) return;
                        uint8_t* base = smem + st * KNN_STAGE_BYTES;
                        mbar_expect_tx(&full_bar[st], KNN_STAGE_BYTES);
                        tma_load_2d(base, &tmA, &full_bar[st], kb * 64, mt * 128);
                        tma_load_2d(base + KNN_A_BYTES, &tmB, &full_bar[st], kb * 64, ct * KNN_BN);
                    }
            }
        }
        return;
    }
    // ======================= consumers: 64 rows per warpgroup, then the selection epilogue =======================
    reg_alloc<CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1, tid_epi = (int)threadIdx.x - 128;
    const int q = lane & 3;
    const int r0 = wg * 64 + 16 * (warp & 3) + (lane >> 2);     // fragment rows r0 and r0 + 8 of the tile (wgmma.cuh)
    static_assert(EPI_THREADS == KNN_BN, "one column-vector entry per consumer thread");
    float acc[KNN_BN / 2];
    int stg = 0;
    for (int t = blockIdx.x; t < items; t += gridDim.x) {
        const int mt = t / p.splits, sp = t % p.splits, c0 = sp * p.per_split;
        const int c1 = min(p.n_tiles, c0 + p.per_split);
        const int row0 = mt * 128 + r0, row1 = row0 + 8;
        const bool ok0 = row0 < p.n_rows, ok1 = row1 < p.n_rows;
        // rows past n_rows (TMA zero fill) get an infinite norm: they never enter a list
        const float na0 = ok0 ? __ldg(p.na + row0) : INFINITY, na1 = ok1 ? __ldg(p.na + row1) : INFINITY;
        float l0[KNN_MAX_K], l1[KNN_MAX_K];
        float thr0 = INFINITY, thr1 = INFINITY;
        bool cv0 = false, cv1 = false;
        int n0 = 0, n1 = 0;
        if constexpr (MODE == KNN_KTH) {
#pragma unroll
            for (int i = 0; i < KNN_MAX_K; ++i) { l0[i] = INFINITY; l1[i] = INFINITY; }
        }
        for (int ct = c0; ct < c1; ++ct) {
            int prev = 0;
            for (int kb = 0; kb < p.kblocks; ++kb, ++stg) {
                const int st = stg % KNN_STAGES;
                if (!mbar_wait(&full_bar[st], (stg / KNN_STAGES) & 1, 12)) return;
                wgmma_fence();
                const uint32_t a_addr = smem_u32(smem + st * KNN_STAGE_BYTES) + (uint32_t)wg * 8192u;
                const uint32_t b_addr = smem_u32(smem + st * KNN_STAGE_BYTES) + KNN_A_BYTES;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_m64n256_f16<0, 0>(acc, wg_smem_desc(a_addr + k * 32, 16, 1024), wg_smem_desc(b_addr + k * 32, 16, 1024),
                                            (kb | k) != 0 ? 1u : 0u);
                wgmma_commit();
                // one group in flight: the previous slab's wgmmas have retired, so its stage goes back to the producer
                wgmma_wait<1>();
                if (kb > 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
                prev = st;
            }
            wgmma_wait<0>();
            wgmma_reg_fence(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            named_bar_sync(1, EPI_THREADS);                  // the previous tile's readers are done with the column vectors
            {
                const int c = tid_epi, col = ct * KNN_BN + c;   // EPI_THREADS == KNN_BN: one column per thread
                const bool valid = col < p.n_cols;
                if constexpr (MODE == KNN_KTH) {
                    s_nb[c] = valid ? __ldg(p.nb + col) : INFINITY;   // masked columns: d2 = inf never enters a list
                } else {
                    const __half r = valid ? p.radii[col] : __float2half(0.f);
                    s_nb[c] = valid ? __ldg(p.nb + col) : 0.f;
                    s_rf[c] = __half2float(r);
                    s_thr[c] = valid ? knn_cover_bound(r) : -1.f;        // masked columns never cover
                }
            }
            named_bar_sync(1, EPI_THREADS);
            if constexpr (MODE == KNN_KTH) {
                const int k1 = p.kk - 1;
#pragma unroll
                for (int j = 0; j < KNN_BN / 8; ++j) {
                    const float2 nb2 = *reinterpret_cast<const float2*>(s_nb + 8 * j + 2 * q);
                    float v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 0], na0 + nb2.x));
                    if (v < thr0) { knn_insert(l0, v); thr0 = knn_at(l0, k1); }
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 1], na0 + nb2.y));
                    if (v < thr0) { knn_insert(l0, v); thr0 = knn_at(l0, k1); }
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 2], na1 + nb2.x));
                    if (v < thr1) { knn_insert(l1, v); thr1 = knn_at(l1, k1); }
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 3], na1 + nb2.y));
                    if (v < thr1) { knn_insert(l1, v); thr1 = knn_at(l1, k1); }
                }
            } else if constexpr (MODE == KNN_COUNT) {
#pragma unroll
                for (int j = 0; j < KNN_BN / 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    const float2 nb2 = *reinterpret_cast<const float2*>(s_nb + c);
                    const float2 th2 = *reinterpret_cast<const float2*>(s_thr + c);
                    float v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 0], na0 + nb2.x));
                    if (v <= th2.x && knn_lt(v, s_rf[c])) ++n0;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 1], na0 + nb2.y));
                    if (v <= th2.y && knn_lt(v, s_rf[c + 1])) ++n0;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 2], na1 + nb2.x));
                    if (v <= th2.x && knn_lt(v, s_rf[c])) ++n1;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 3], na1 + nb2.y));
                    if (v <= th2.y && knn_lt(v, s_rf[c + 1])) ++n1;
                }
            } else {
#pragma unroll
                for (int j = 0; j < KNN_BN / 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    const float2 nb2 = *reinterpret_cast<const float2*>(s_nb + c);
                    const float2 th2 = *reinterpret_cast<const float2*>(s_thr + c);
                    float v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 0], na0 + nb2.x));
                    if (v <= th2.x && knn_le(v, s_rf[c])) cv0 = true;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 1], na0 + nb2.y));
                    if (v <= th2.y && knn_le(v, s_rf[c + 1])) cv0 = true;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 2], na1 + nb2.x));
                    if (v <= th2.x && knn_le(v, s_rf[c])) cv1 = true;
                    v = fmaxf(0.f, fmaf(-2.f, acc[4 * j + 3], na1 + nb2.y));
                    if (v <= th2.y && knn_le(v, s_rf[c + 1])) cv1 = true;
                }
            }
        }
        // merge over the quad of lanes that share the two rows, then one lane writes this split's entry of each row
        if constexpr (MODE == KNN_KTH) {
#pragma unroll
            for (int m = 1; m <= 2; m <<= 1) {
                float o0[KNN_MAX_K], o1[KNN_MAX_K];
#pragma unroll
                for (int i = 0; i < KNN_MAX_K; ++i) { o0[i] = __shfl_xor_sync(0xffffffffu, l0[i], m); o1[i] = __shfl_xor_sync(0xffffffffu, l1[i], m); }
#pragma unroll
                for (int i = 0; i < KNN_MAX_K; ++i) { knn_insert(l0, o0[i]); knn_insert(l1, o1[i]); }
            }
            if (q == 0) {
                float* d0 = p.part + ((size_t)sp * p.n_rows + row0) * p.kk;
                float* d1 = d0 + (size_t)8 * p.kk;
#pragma unroll
                for (int i = 0; i < KNN_MAX_K; ++i) {
                    if (i < p.kk) { if (ok0) d0[i] = l0[i]; if (ok1) d1[i] = l1[i]; }
                }
            }
        } else if constexpr (MODE == KNN_COUNT) {
            n0 += __shfl_xor_sync(0xffffffffu, n0, 1); n0 += __shfl_xor_sync(0xffffffffu, n0, 2);
            n1 += __shfl_xor_sync(0xffffffffu, n1, 1); n1 += __shfl_xor_sync(0xffffffffu, n1, 2);
            if (q == 0) {
                int* d = p.counts + (size_t)sp * p.n_rows;
                if (ok0) d[row0] = n0;
                if (ok1) d[row1] = n1;
            }
        } else {
            int f0 = cv0 ? 1 : 0, f1 = cv1 ? 1 : 0;
            f0 |= __shfl_xor_sync(0xffffffffu, f0, 1); f0 |= __shfl_xor_sync(0xffffffffu, f0, 2);
            f1 |= __shfl_xor_sync(0xffffffffu, f1, 1); f1 |= __shfl_xor_sync(0xffffffffu, f1, 2);
            if (q == 0) {
                uint8_t* d = p.flags + (size_t)sp * p.n_rows;
                if (ok0) d[row0] = (uint8_t)f0;
                if (ok1) d[row1] = (uint8_t)f1;
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
knn_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const KnnParams p) {
    knn_wgmma_body<MODE>(tmA, tmB, p);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
knn_count_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const KnnParams p) {
    knn_wgmma_body<KNN_COUNT>(tmA, tmB, p);
}

// squared row norms in fp32, one warp per row: lane l sums chunks l, l + 32, ... of 8 elements in order, then a fixed butterfly
__global__ void k_knn_norms(const __half* x, int n, long long ld, int D, float* out) {
    pdl_entry();
    const int row = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    const __half* r = x + (long long)row * ld;
    float s = 0.f;
    for (int c = lane * 8; c < D; c += 256) {
        if (c + 8 <= D) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(r + c));
            const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); s = fmaf(f.x, f.x, s); s = fmaf(f.y, f.y, s); }
        } else {
            for (int e = c; e < D; ++e) { const float f = __half2float(r[e]); s = fmaf(f, f, s); }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[row] = s;
}

// kth: the kk smallest over all splits of a row, then fp16_rn(sqrt_rn(.)) of the kk-th
__global__ void k_knn_kth_final(const float* part, int splits, int n_rows, int kk, __half* out) {
    pdl_entry();
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    float l[KNN_MAX_K];
#pragma unroll
    for (int i = 0; i < KNN_MAX_K; ++i) l[i] = INFINITY;
    for (int s = 0; s < splits; ++s) {
        const float* src = part + ((size_t)s * n_rows + row) * kk;
        for (int i = 0; i < kk; ++i) knn_insert(l, src[i]);
    }
    out[row] = __float2half_rn(__fsqrt_rn(knn_at(l, kk - 1)));
}

// cover: OR over the splits
__global__ void k_knn_cover_final(const uint8_t* flags, int splits, int n_rows, uint8_t* out) {
    pdl_entry();
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    uint8_t f = 0;
    for (int s = 0; s < splits; ++s) f |= flags[(size_t)s * n_rows + row];
    out[row] = f;
}

// count: sum over the splits
__global__ void k_knn_count_final(const int* counts, int splits, int n_rows, int* out) {
    pdl_entry();
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    int c = 0;
    for (int s = 0; s < splits; ++s) c += counts[(size_t)s * n_rows + row];
    out[row] = c;
}

// ------------------------------------------------------------------------------------------------ host side
struct KnnPlan {
    int m_tiles = 0, n_tiles = 0, splits = 1, per_split = 0, kblocks = 0;
    size_t off_nb = 0, off_part = 0, total = 0;
};
inline size_t knn_align(size_t n) { return (n + 255) & ~size_t(255); }
// Column splits: the fewest waves of (row tile, column range) items over kPlanSms CTAs, counted in column tiles per CTA; among
// equal counts the largest split up to max(16, SMs / row tiles), so that CTAs running together share a row tile.  Fixed by the
// shape alone (kPlanSms, not the device), so the scratch size is too; the result does not depend on it.
inline KnnPlan knn_plan(KnnMode mode, int n_rows, int n_cols, int D, int kk) {
    KnnPlan pl;
    pl.m_tiles = (n_rows + 127) / 128; pl.n_tiles = (n_cols + KNN_BN - 1) / KNN_BN; pl.kblocks = (D + 63) / 64;
    const int cap = std::min(pl.n_tiles, std::max(16, (kPlanSms + pl.m_tiles - 1) / pl.m_tiles));
    long long best = -1;
    for (int s = 1; s <= cap; ++s) {
        const int per = (pl.n_tiles + s - 1) / s;
        const long long items = (long long)pl.m_tiles * ((pl.n_tiles + per - 1) / per);
        const long long cost = (items + kPlanSms - 1) / kPlanSms * per;
        if (best < 0 || cost <= best) { best = cost; pl.splits = s; }
    }
    pl.per_split = (pl.n_tiles + pl.splits - 1) / pl.splits;
    pl.splits = (pl.n_tiles + pl.per_split - 1) / pl.per_split;   // no empty ranges
    pl.off_nb = knn_align((size_t)n_rows * 4);
    pl.off_part = pl.off_nb + knn_align((size_t)n_cols * 4);
    const size_t entry = mode == KNN_KTH ? (size_t)kk * 4 : mode == KNN_COUNT ? 4 : 1;
    const size_t part = (size_t)pl.splits * n_rows * entry;
    pl.total = pl.off_part + knn_align(part);
    return pl;
}

// fp16 matrix [rows][ld] viewed as (D, rows), box 64 x box_rows, 128-byte swizzle; columns past D and rows past `rows` read as 0
inline int make_tmap_f16_2d(CUtensorMap* m, const void* ptr, int D, int rows, long long ld, int box_rows) {
    auto fn = tmap_encode_fn();
    if (!fn) return fail(-3, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(-5, "cuTensorMapEncodeTiled(fp16 2d) failed: %d (D=%d rows=%d ld=%lld)", (int)r, D, rows, ld);
    return 0;
}

// Every pass: norms of rows and columns, the wgmma pass, the finalise.  KNN_KTH: kth radii into out (fp16 [n_rows]);
// KNN_COVER: coverage flags of the rows against radii (u8 [n_rows]); KNN_COUNT: counts of the balls holding each row (int32
// [n_rows]).  Arguments are checked by the caller.
inline int knn_launch(KnnMode mode, const __half* rows, int n_rows, long long ld_r, const __half* cols, int n_cols, long long ld_c,
                      int D, int kk, const __half* radii, void* out, void* scratch, cudaStream_t st) {
    const KnnPlan pl = knn_plan(mode, n_rows, n_cols, D, kk);
    uint8_t* s = static_cast<uint8_t*>(scratch);
    KnnParams p;
    p.n_rows = n_rows; p.n_cols = n_cols; p.kblocks = pl.kblocks; p.m_tiles = pl.m_tiles; p.n_tiles = pl.n_tiles;
    p.splits = pl.splits; p.per_split = pl.per_split; p.kk = kk;
    p.na = reinterpret_cast<float*>(s); p.nb = reinterpret_cast<float*>(s + pl.off_nb); p.radii = radii;
    p.part = mode == KNN_KTH ? reinterpret_cast<float*>(s + pl.off_part) : nullptr;
    p.flags = mode == KNN_COVER ? s + pl.off_part : nullptr;
    p.counts = mode == KNN_COUNT ? reinterpret_cast<int*>(s + pl.off_part) : nullptr;
    CUtensorMap tA, tB;
    int rc = make_tmap_f16_2d(&tA, rows, D, n_rows, ld_r, 128);
    if (!rc) rc = make_tmap_f16_2d(&tB, cols, D, n_cols, ld_c, KNN_BN);
    if (rc) return rc;
    launch_k(k_knn_norms, (unsigned)((n_rows + 7) / 8), 256, 0, st, rows, n_rows, ld_r, D, const_cast<float*>(p.na));
    launch_k(k_knn_norms, (unsigned)((n_cols + 7) / 8), 256, 0, st, cols, n_cols, ld_c, D, const_cast<float*>(p.nb));
    DDPM_CUDA_OK(cudaGetLastError());
    int dev = 0, sms = 0;
    DDPM_CUDA_OK(cudaGetDevice(&dev));
    DDPM_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int items = pl.m_tiles * pl.splits;
    const int ctas = std::max(1, std::min(items, sms));
    auto kern = mode == KNN_KTH ? knn_wgmma_kernel<KNN_KTH> : mode == KNN_COVER ? knn_wgmma_kernel<KNN_COVER> : knn_count_kernel;
    DDPM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, KNN_SMEM));
    launch_k(kern, ctas, GEMM_THREADS, KNN_SMEM, st, tA, tB, p);
    DDPM_CUDA_OK(cudaGetLastError());
    const unsigned g = (unsigned)((n_rows + 255) / 256);
    if (mode == KNN_KTH) launch_k(k_knn_kth_final, g, 256, 0, st, (const float*)p.part, pl.splits, n_rows, kk, static_cast<__half*>(out));
    else if (mode == KNN_COVER) launch_k(k_knn_cover_final, g, 256, 0, st, (const uint8_t*)p.flags, pl.splits, n_rows, static_cast<uint8_t*>(out));
    else launch_k(k_knn_count_final, g, 256, 0, st, (const int*)p.counts, pl.splits, n_rows, static_cast<int*>(out));
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace ddpm
