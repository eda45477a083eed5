// The 2-D toy denoiser of ddpm_torch/toy (toy_model.py: Decoder) on wgmma: forward, training loss, backward, the fixed-order
// gradient reduce and the whole ancestral sampler chain in one launch.
//
// Model (M = mid_features in {64, 128}, D = in_features in 1..4, L = num_temporal_layers >= 1, ONE TemporalLayer applied L times):
//   e = lrelu(t_proj(emb(t)))              E = enc(e)  (the same for every application, so computed once per row)
//   h = in_fc(x);  L x { u = fc1(lrelu(LN1(h))) + E;  h = fc2(lrelu(LN2(u))) + h };  out = out_fc(LN_out(h))
// LayerNorm eps 1e-5 (affine), LeakyReLU slope 0.02; fc1 / fc2 / in_fc have no bias.
//
// Every kernel is one warpgroup per CTA (128 threads) that owns 64-row tiles, persistent over the tiles.  A [64 x M] activation lives
// in the wgmma accumulator fragment (wgmma.cuh); LayerNorm statistics use the in-thread + lane-quad reduction of the attention
// softmax; the bf16 operand of the next GEMM goes back to shared memory in the K-major 128-byte swizzled layout.  The weights are
// staged once per CTA, converted from the fp32 master parameters to bf16 on the way (no packed copy: a kernel always reads the
// current values).  A weight tile W[out][in] serves as the K-major B operand of Y = A W^T and, read MN-major, of dA = dY W.
// in_fc (K = D) and out_fc (N = D) run on CUDA cores.
//
// Launches:
//   toy_temb_kernel      rows -> E [rows][M] fp32 (t_proj + enc on the tensor cores); the sampler calls it with rows = steps
//   toy_fwd_kernel       x (or q_sample(x_0, t, noise)) -> out, optional per-row mse loss; training saves h_l, u_l, x_t, out
//   toy_bwd_kernel       d_out (or the per-row loss gradient) -> dx, dE = sum over layers of du, per-CTA weight-gradient partials
//   toy_temb_bwd_kernel  dE -> partials of enc and t_proj
//   toy_reduce_kernel    partials -> flat fp32 gradient in parameters() order, summed in a fixed order (no atomics)
//   toy_sample_kernel    all S steps of p_sample for the CTA's rows, x in registers
// The backward reads the activations the training forward saved (h_l and u_l per layer, fp32) rather than recomputing the forward:
// at B = 1000 they are 3.5 MB, and the recompute would double the backward's GEMMs.
#pragma once
#include "ptx.cuh"
#include "wgmma.cuh"
#include "../../include/ddpm_b200.h"

namespace ddpm {

constexpr int TOY_THREADS = 128;
constexpr float TOY_SLOPE = 0.02f, TOY_LN_EPS = 1e-5f;
constexpr int TOY_FWD_CTAS = 264, TOY_BWD_CTAS = 132;     // fwd / sampler: two CTAs per SM; bwd: one partial slot per CTA

// flat-gradient offsets of the 15 parameters, parameters() order
struct ToyLayout {
    int M, D, L;
    long long in_w, n1_g, n1_b, fc1, n2_g, n2_b, fc2, enc_w, enc_b, on_g, on_b, out_w, out_b, tp_w, tp_b, P, Pp;
    __host__ __device__ ToyLayout(int M_, int D_, int L_) : M(M_), D(D_), L(L_) {
        long long o = 0;
        in_w = o; o += (long long)M * D; n1_g = o; o += M; n1_b = o; o += M; fc1 = o; o += (long long)M * M;
        n2_g = o; o += M; n2_b = o; o += M; fc2 = o; o += (long long)M * M; enc_w = o; o += (long long)M * M; enc_b = o; o += M;
        on_g = o; o += M; on_b = o; o += M; out_w = o; o += (long long)D * M; out_b = o; o += D; tp_w = o; o += (long long)M * M;
        tp_b = o; o += M; P = o; Pp = (o + 63) & ~63LL;
    }
};

struct ToyArgs {
    ddpm_toy_params w;
    int M, D, L, B;
    const float* x;              // fwd: x [B][D]; sampler: x in/out
    const long long* t;          // per-row timesteps (temb); null: t = row index (the sampler's step table)
    const float* x0; const float* noise; const float* sa; const float* s1a;     // q_sample / loss
    float* out; float* loss;
    float* E;                    // [rows][M]
    float* h_sv; float* u_sv; float* x_sv; float* out_sv;                      // training saves
    const float* d_out; const float* g;                                        // backward seeds (one of them)
    float* dx; float* dE; float* part;                                         // backward outputs
    const float* coef; const float* z; int S;                                  // sampler
};

__device__ __forceinline__ float toy_lrelu(float v) { return v > 0.f ? v : v * TOY_SLOPE; }
__device__ __forceinline__ float toy_lrelu_grad(float v) { return v > 0.f ? 1.f : TOY_SLOPE; }

// byte offset of element (row R, column c) in a K-major SWIZZLE_128B bf16 tile of `rows` rows (64-column slabs of rows x 128 B)
__device__ __forceinline__ uint32_t toy_off(int rows, int R, int c) {
    return (uint32_t)((c >> 6) * rows * 128 + R * 128 + ((((c & 63) >> 3) ^ (R & 7)) << 4) + (c & 7) * 2);
}

// fp32 [rows][M] row-major (global) -> bf16 swizzled tile
__device__ __forceinline__ void toy_stage_w(uint8_t* tile, const float* __restrict__ W, int rows, int M) {
    const int chunks = rows * M / 8;
    for (int i = threadIdx.x; i < chunks; i += TOY_THREADS) {
        const int r = i / (M / 8), c0 = (i % (M / 8)) * 8;
        const float4 a = __ldg(reinterpret_cast<const float4*>(W + (size_t)r * M + c0));
        const float4 b = __ldg(reinterpret_cast<const float4*>(W + (size_t)r * M + c0 + 4));
        st_shared_v4(tile + toy_off(rows, r, c0), pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
    }
}

__device__ __forceinline__ void toy_sync_for_wgmma() { fence_proxy_async_smem(); __syncthreads(); }

// Y = A W^T: A = 64-row activation tile (K-major), W = [M out][M in] tile (K-major B); scale_d = 0 overwrites, 1 accumulates
template <int M>
__device__ __forceinline__ void toy_mm_nt(float (&d)[M / 2], const uint8_t* A, const uint8_t* W, uint32_t scale_d) {
    const uint32_t a = smem_u32(A), b = smem_u32(W);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < M / 64; ++kc)
#pragma unroll
        for (int k = 0; k < 4; ++k)
            Wgmma<M>::template mma<0, 0>(d, wg_smem_desc(a + kc * 8192 + k * 32, 16, 1024), wg_smem_desc(b + kc * M * 128 + k * 32, 16, 1024),
                                        (kc | k) ? 1u : scale_d);
    wgmma_commit(); wgmma_wait<0>(); wgmma_reg_fence(d);
}
// dA = dY W: dY tile K-major (K = out), W read MN-major (K rows = out, 64-column MN blocks = in slabs)
template <int M>
__device__ __forceinline__ void toy_mm_nn(float (&d)[M / 2], const uint8_t* dY, const uint8_t* W) {
    const uint32_t a = smem_u32(dY), b = smem_u32(W);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < M / 64; ++kc)
#pragma unroll
        for (int k = 0; k < 4; ++k)
            Wgmma<M>::template mma<0, 1>(d, wg_smem_desc(a + kc * 8192 + k * 32, 16, 1024), wg_smem_desc(b + (kc * 64 + k * 16) * 128, M * 128, 1024),
                                        (kc | k) ? 1u : 0u);
    wgmma_commit(); wgmma_wait<0>(); wgmma_reg_fence(d);
}
// dW[out][in] partial over the tile's 64 rows = dY^T A, both operands MN-major (rows are K); one m64 block of outputs per call,
// added into the CTA's fp32 partial slot (no other CTA touches it)
template <int M>
__device__ __forceinline__ void toy_mm_wgrad(float (&d)[M / 2], const uint8_t* dY, const uint8_t* A, float* __restrict__ slot) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int mb = 0; mb < M / 64; ++mb) {
        const uint32_t a = smem_u32(dY) + mb * 8192, b = smem_u32(A);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
            Wgmma<M>::template mma<1, 1>(d, wg_smem_desc(a + k * 2048, 8192, 1024), wg_smem_desc(b + k * 2048, 8192, 1024), k ? 1u : 0u);
        wgmma_commit(); wgmma_wait<0>(); wgmma_reg_fence(d);
        const int r0 = mb * 64 + 16 * w + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < M / 8; ++j) {
            float* p0 = slot + (size_t)r0 * M + 8 * j + cq;       // scalar: a slot offset is odd when in_features is
            float* p1 = slot + (size_t)(r0 + 8) * M + 8 * j + cq;
            p0[0] += d[4 * j]; p0[1] += d[4 * j + 1]; p1[0] += d[4 * j + 2]; p1[1] += d[4 * j + 3];
        }
    }
}

// fragment -> bf16 tile (through f)
template <int M, typename F>
__device__ __forceinline__ void toy_put(uint8_t* tile, F f) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int R0 = 16 * w + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < M / 8; ++j) {
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(tile + toy_off(64, R0, 8 * j + cq))), "r"(pack_bf16x2(f(4 * j), f(4 * j + 1))) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(tile + toy_off(64, R0 + 8, 8 * j + cq))), "r"(pack_bf16x2(f(4 * j + 2), f(4 * j + 3))) : "memory");
    }
}

__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// LayerNorm row statistics of the fragment's two rows: mean and 1/sqrt(var + eps), two-pass
template <int M>
__device__ __forceinline__ void toy_ln_stats(const float (&d)[M / 2], float (&mean)[2], float (&rstd)[2]) {
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < M / 8; ++j) { s0 += d[4 * j] + d[4 * j + 1]; s1 += d[4 * j + 2] + d[4 * j + 3]; }
    mean[0] = quad_sum(s0) * (1.f / M); mean[1] = quad_sum(s1) * (1.f / M);
    float q0 = 0.f, q1 = 0.f;
#pragma unroll
    for (int j = 0; j < M / 8; ++j) {
        const float a = d[4 * j] - mean[0], b = d[4 * j + 1] - mean[0], c = d[4 * j + 2] - mean[1], e = d[4 * j + 3] - mean[1];
        q0 += a * a + b * b; q1 += c * c + e * e;
    }
    rstd[0] = rsqrtf(quad_sum(q0) * (1.f / M) + TOY_LN_EPS); rstd[1] = rsqrtf(quad_sum(q1) * (1.f / M) + TOY_LN_EPS);
}

// column of fragment element i (i = 4j + q): 8j + 2(lane%4) + (q&1); row half q>>1
__device__ __forceinline__ int toy_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

// Column sums over the tile's 64 rows of f(i) added into dst[0..M): lane-group shuffles, then the four warps in order through smem.
template <int M, typename F>
__device__ __forceinline__ void toy_colsum(float* red, float* __restrict__ dst, F f) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float s[M / 4];
#pragma unroll
    for (int j = 0; j < M / 8; ++j) { s[2 * j] = f(4 * j) + f(4 * j + 2); s[2 * j + 1] = f(4 * j + 1) + f(4 * j + 3); }
#pragma unroll
    for (int i = 0; i < M / 4; ++i) {
        s[i] += __shfl_xor_sync(0xffffffffu, s[i], 4); s[i] += __shfl_xor_sync(0xffffffffu, s[i], 8); s[i] += __shfl_xor_sync(0xffffffffu, s[i], 16);
    }
    if (lane < 4)
#pragma unroll
        for (int j = 0; j < M / 8; ++j) { red[w * M + 8 * j + 2 * lane] = s[2 * j]; red[w * M + 8 * j + 2 * lane + 1] = s[2 * j + 1]; }
    __syncthreads();
    if (threadIdx.x < M) dst[threadIdx.x] += ((red[threadIdx.x] + red[M + threadIdx.x]) + red[2 * M + threadIdx.x]) + red[3 * M + threadIdx.x];
    __syncthreads();
}

// small fp32 parameters staged per CTA: LN gamma/beta x3, in_fc [M][4], out_fc [4][M], out_b [4]
template <int M> struct ToySmall {
    float n1g[M], n1b[M], n2g[M], n2b[M], ong[M], onb[M], in_w[M][4], out_w[4][M], out_b[4];
};
template <int M>
__device__ __forceinline__ void toy_stage_small(ToySmall<M>* s, const ToyArgs& a) {
    for (int c = threadIdx.x; c < M; c += TOY_THREADS) {
        s->n1g[c] = a.w.norm1_weight[c]; s->n1b[c] = a.w.norm1_bias[c]; s->n2g[c] = a.w.norm2_weight[c]; s->n2b[c] = a.w.norm2_bias[c];
        s->ong[c] = a.w.out_norm_weight[c]; s->onb[c] = a.w.out_norm_bias[c];
#pragma unroll
        for (int d = 0; d < 4; ++d) { s->in_w[c][d] = d < a.D ? a.w.in_fc_weight[c * a.D + d] : 0.f; s->out_w[d][c] = d < a.D ? a.w.out_fc_weight[d * M + c] : 0.f; }
    }
    if (threadIdx.x < 4) s->out_b[threadIdx.x] = (int)threadIdx.x < a.D ? a.w.out_fc_bias[threadIdx.x] : 0.f;
}

template <int M> struct ToyFwdSmem {
    uint8_t fc1[M * M * 2], fc2[M * M * 2], ta[64 * M * 2], tb[64 * M * 2];
    ToySmall<M> s;
    float red[4 * M];
};

// in_fc on CUDA cores: h(r, c) = sum_d x(r, d) W_in(c, d)
template <int M>
__device__ __forceinline__ void toy_in_fc(float (&h)[M / 2], const float (&x)[2][4], const ToySmall<M>* s) {
#pragma unroll
    for (int i = 0; i < M / 2; ++i) {
        const int c = toy_col(i), r = (i >> 1) & 1;
        h[i] = ((x[r][0] * s->in_w[c][0] + x[r][1] * s->in_w[c][1]) + x[r][2] * s->in_w[c][2]) + x[r][3] * s->in_w[c][3];
    }
}

// one TemporalLayer on the fragment h (residual accumulated by the fc2 wgmma); E(i) gives enc(e) at fragment element i.
// When u_save is set, writes u (pre-LN2) of the two rows.
template <int M, typename EF>
__device__ __forceinline__ void toy_layer(float (&h)[M / 2], float (&u)[M / 2], ToyFwdSmem<M>* sm, EF E) {
    float mean[2], rstd[2];
    toy_ln_stats<M>(h, mean, rstd);
    __syncthreads();
    toy_put<M>(sm->ta, [&](int i) { const int c = toy_col(i), r = (i >> 1) & 1; return toy_lrelu((h[i] - mean[r]) * rstd[r] * sm->s.n1g[c] + sm->s.n1b[c]); });
    toy_sync_for_wgmma();
#pragma unroll
    for (int i = 0; i < M / 2; ++i) u[i] = E(i);
    toy_mm_nt<M>(u, sm->ta, sm->fc1, 1u);
    toy_ln_stats<M>(u, mean, rstd);
    toy_put<M>(sm->tb, [&](int i) { const int c = toy_col(i), r = (i >> 1) & 1; return toy_lrelu((u[i] - mean[r]) * rstd[r] * sm->s.n2g[c] + sm->s.n2b[c]); });
    toy_sync_for_wgmma();
    toy_mm_nt<M>(h, sm->tb, sm->fc2, 1u);
}

// out_fc(LN_out(h)) on CUDA cores; every lane of a quad ends with out[2][4] of its two rows
template <int M>
__device__ __forceinline__ void toy_head(const float (&h)[M / 2], const ToySmall<M>* s, float (&out)[2][4]) {
    float mean[2], rstd[2];
    toy_ln_stats<M>(h, mean, rstd);
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int d = 0; d < 4; ++d) out[r][d] = 0.f;
#pragma unroll
    for (int i = 0; i < M / 2; ++i) {
        const int c = toy_col(i), r = (i >> 1) & 1;
        const float n = (h[i] - mean[r]) * rstd[r] * s->ong[c] + s->onb[c];
#pragma unroll
        for (int d = 0; d < 4; ++d) out[r][d] += n * s->out_w[d][c];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int d = 0; d < 4; ++d) out[r][d] = quad_sum(out[r][d]) + s->out_b[d];
}

__device__ __forceinline__ int toy_tiles(int B) { return (B + 63) / 64; }

// ------------------------------------------------------------------------------------------------ timestep path
template <int M> struct ToyTembSmem { uint8_t tp[M * M * 2], enc[M * M * 2], ta[64 * M * 2], tb[64 * M * 2], td[64 * M * 2]; float red[4 * M]; };

// sinusoidal embedding (k_timestep_embedding's arithmetic) of the tile's rows -> bf16 tile
template <int M>
__device__ __forceinline__ void toy_put_emb(uint8_t* tile, const long long* t, int row0, int rows) {
    constexpr int half = M / 2;
    const float k = logf(10000.f) / (float)(half - 1);
    for (int i = threadIdx.x; i < 64 * half; i += TOY_THREADS) {
        const int R = i / half, j = i % half, g = row0 + R;
        const float tv = g < rows ? (float)(t ? t[g] : (long long)g) : 0.f;
        const float a = tv * expf(-(float)j * k);
        *reinterpret_cast<__nv_bfloat16*>(tile + toy_off(64, R, j)) = __float2bfloat16_rn(sinf(a));
        *reinterpret_cast<__nv_bfloat16*>(tile + toy_off(64, R, half + j)) = __float2bfloat16_rn(cosf(a));
    }
}

// pre = emb(t) t_proj^T + b into d; e = lrelu(pre) -> tile tb
template <int M>
__device__ __forceinline__ void toy_temb_tile(float (&d)[M / 2], ToyTembSmem<M>* sm, const ToyArgs& a, int row0, int rows) {
    __syncthreads();
    toy_put_emb<M>(sm->ta, a.t, row0, rows);
    toy_sync_for_wgmma();
    toy_mm_nt<M>(d, sm->ta, sm->tp, 0u);
#pragma unroll
    for (int i = 0; i < M / 2; ++i) d[i] += __ldg(a.w.t_proj_bias + toy_col(i));
    toy_put<M>(sm->tb, [&](int i) { return toy_lrelu(d[i]); });
    toy_sync_for_wgmma();
}

template <int M>
__global__ void __launch_bounds__(TOY_THREADS) toy_temb_kernel(const ToyArgs a, int rows) {
    pdl_entry();
    extern __shared__ uint8_t smem_raw[];
    auto* sm = reinterpret_cast<ToyTembSmem<M>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    toy_stage_w(sm->tp, a.w.t_proj_weight, M, M);
    toy_stage_w(sm->enc, a.w.enc_weight, M, M);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float d[M / 2];
    for (int tile = blockIdx.x; tile < toy_tiles(rows); tile += gridDim.x) {
        const int row0 = tile * 64;
        toy_temb_tile<M>(d, sm, a, row0, rows);
        toy_mm_nt<M>(d, sm->tb, sm->enc, 0u);
        const int g0 = row0 + 16 * w + (lane >> 2);
#pragma unroll
        for (int i = 0; i < M / 2; ++i) {
            const int c = toy_col(i), g = g0 + 8 * ((i >> 1) & 1);
            if (g < rows) a.E[(size_t)g * M + c] = d[i] + __ldg(a.w.enc_bias + c);
        }
    }
}

// ------------------------------------------------------------------------------------------------ forward
template <int M>
__global__ void __launch_bounds__(TOY_THREADS) toy_fwd_kernel(const ToyArgs a) {
    pdl_entry();
    extern __shared__ uint8_t smem_raw[];
    auto* sm = reinterpret_cast<ToyFwdSmem<M>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    toy_stage_w(sm->fc1, a.w.fc1_weight, M, M);
    toy_stage_w(sm->fc2, a.w.fc2_weight, M, M);
    toy_stage_small<M>(&sm->s, a);
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, q = lane & 3;
    const int D = a.D, B = a.B;
    float h[M / 2], u[M / 2];
    for (int tile = blockIdx.x; tile < toy_tiles(B); tile += gridDim.x) {
        const int g0 = tile * 64 + 16 * w + (lane >> 2);
        const int gr[2] = {g0, g0 + 8};
        float x[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int d = 0; d < 4; ++d) {
                float v = 0.f;
                if (gr[r] < B && d < D) {
                    if (a.x0) {            // q_sample: coef1 * x_0 + coef2 * noise (toy/diffusion.py:9-14), no contraction
                        const long long tt = a.t[gr[r]];
                        v = __fadd_rn(__fmul_rn(a.sa[tt], a.x0[(size_t)gr[r] * D + d]), __fmul_rn(a.s1a[tt], a.noise[(size_t)gr[r] * D + d]));
                    } else v = a.x[(size_t)gr[r] * D + d];
                }
                x[r][d] = v;
            }
        if (a.x_sv && q < D)
#pragma unroll
            for (int r = 0; r < 2; ++r) if (gr[r] < B) a.x_sv[(size_t)gr[r] * D + q] = x[r][q];
        toy_in_fc<M>(h, x, &sm->s);
        for (int l = 0; l < a.L; ++l) {
            if (a.h_sv)
#pragma unroll
                for (int i = 0; i < M / 2; i += 2) {
                    const int g = gr[(i >> 1) & 1];
                    if (g < B) *reinterpret_cast<float2*>(a.h_sv + ((size_t)l * B + g) * M + toy_col(i)) = make_float2(h[i], h[i + 1]);
                }
            toy_layer<M>(h, u, sm, [&](int i) { const int g = gr[(i >> 1) & 1]; return g < B ? a.E[(size_t)g * M + toy_col(i)] : 0.f; });
            if (a.u_sv)
#pragma unroll
                for (int i = 0; i < M / 2; i += 2) {
                    const int g = gr[(i >> 1) & 1];
                    if (g < B) *reinterpret_cast<float2*>(a.u_sv + ((size_t)l * B + g) * M + toy_col(i)) = make_float2(u[i], u[i + 1]);
                }
        }
        if (a.h_sv)
#pragma unroll
            for (int i = 0; i < M / 2; i += 2) {
                const int g = gr[(i >> 1) & 1];
                if (g < B) *reinterpret_cast<float2*>(a.h_sv + ((size_t)a.L * B + g) * M + toy_col(i)) = make_float2(h[i], h[i + 1]);
            }
        float o[2][4];
        toy_head<M>(h, &sm->s, o);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (gr[r] >= B) continue;
            if (q < D) {
                if (a.out) a.out[(size_t)gr[r] * D + q] = o[r][q];
                if (a.out_sv) a.out_sv[(size_t)gr[r] * D + q] = o[r][q];
            }
            if (a.loss && q == 0) {     // mean((noise - out)^2) over the D features
                float s = 0.f;
                for (int d = 0; d < D; ++d) { const float e = a.noise[(size_t)gr[r] * D + d] - o[r][d]; s += e * e; }
                a.loss[gr[r]] = s / (float)D;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward
template <int M> struct ToyBwdSmem {
    uint8_t fc1[M * M * 2], fc2[M * M * 2], ta[64 * M * 2], tb[64 * M * 2];
    ToySmall<M> s;
    float red[4 * M];
};

// dv = rstd * (gy - mean(gy) - xhat * mean(gy * xhat)) with gy = dy * gamma (rows of the fragment)
template <int M>
__device__ __forceinline__ void toy_ln_bwd(float (&gy)[M / 2], const float (&xh)[M / 2], const float (&rstd)[2]) {
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll
    for (int j = 0; j < M / 8; ++j) {
        a0 += gy[4 * j] + gy[4 * j + 1]; a1 += gy[4 * j + 2] + gy[4 * j + 3];
        b0 += gy[4 * j] * xh[4 * j] + gy[4 * j + 1] * xh[4 * j + 1]; b1 += gy[4 * j + 2] * xh[4 * j + 2] + gy[4 * j + 3] * xh[4 * j + 3];
    }
    a0 = quad_sum(a0) * (1.f / M); a1 = quad_sum(a1) * (1.f / M); b0 = quad_sum(b0) * (1.f / M); b1 = quad_sum(b1) * (1.f / M);
#pragma unroll
    for (int i = 0; i < M / 2; ++i) {
        const int r = (i >> 1) & 1;
        gy[i] = (r ? rstd[1] : rstd[0]) * (gy[i] - (r ? a1 : a0) - xh[i] * (r ? b1 : b0));
    }
}

template <int M>
__global__ void __launch_bounds__(TOY_THREADS) toy_bwd_kernel(const ToyArgs a) {
    pdl_entry();
    extern __shared__ uint8_t smem_raw[];
    auto* sm = reinterpret_cast<ToyBwdSmem<M>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    toy_stage_w(sm->fc1, a.w.fc1_weight, M, M);
    toy_stage_w(sm->fc2, a.w.fc2_weight, M, M);
    toy_stage_small<M>(&sm->s, a);
    __syncthreads();
    const ToyLayout lay(M, a.D, a.L);
    float* slot = a.part + (size_t)blockIdx.x * lay.Pp;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, q = lane & 3;
    const int D = a.D, B = a.B;
    float dh[M / 2], acc[M / 2], xh[M / 2];
    for (int tile = blockIdx.x; tile < toy_tiles(B); tile += gridDim.x) {
        const int g0 = tile * 64 + 16 * w + (lane >> 2);
        const int gr[2] = {g0, g0 + 8};
        auto ld = [&](const float* base, int i) { const int g = gr[(i >> 1) & 1]; return g < B ? base[(size_t)g * M + toy_col(i)] : 0.f; };
        // d_out of the two rows (quad-replicated)
        float dout[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int d = 0; d < 4; ++d) {
                float v = 0.f;
                if (gr[r] < B && d < D) {
                    const size_t k = (size_t)gr[r] * D + d;
                    v = a.g ? a.g[gr[r]] * 2.f * (a.out_sv[k] - a.noise[k]) / (float)D : a.d_out[k];
                }
                dout[r][d] = v;
            }
        // head: n = LN_out(h_L); out = n W_out^T + b
        const float* hL = a.h_sv + (size_t)a.L * B * M;
#pragma unroll
        for (int i = 0; i < M / 2; ++i) acc[i] = ld(hL, i);
        float mean[2], rstd[2];
        toy_ln_stats<M>(acc, mean, rstd);
#pragma unroll
        for (int i = 0; i < M / 2; ++i) { const int r = (i >> 1) & 1; xh[i] = (acc[i] - mean[r]) * rstd[r]; }
        for (int d = 0; d < D; ++d)
            toy_colsum<M>(sm->red, slot + lay.out_w + (size_t)d * M, [&](int i) {
                const int c = toy_col(i), r = (i >> 1) & 1; return dout[r][d] * (xh[i] * sm->s.ong[c] + sm->s.onb[c]); });
        if (threadIdx.x == 0)       // out_fc.bias: the d_out rows summed in row order (the thread reads them from global)
            for (int d = 0; d < D; ++d) {
                float s = 0.f;
                for (int g = tile * 64; g < min(B, tile * 64 + 64); ++g)
                    s += a.g ? a.g[g] * 2.f * (a.out_sv[(size_t)g * D + d] - a.noise[(size_t)g * D + d]) / (float)D : a.d_out[(size_t)g * D + d];
                slot[lay.out_b + d] += s;
            }
#pragma unroll
        for (int i = 0; i < M / 2; ++i) {     // d n
            const int c = toy_col(i), r = (i >> 1) & 1;
            float v = 0.f;
#pragma unroll
            for (int d = 0; d < 4; ++d) v += dout[r][d] * sm->s.out_w[d][c];
            dh[i] = v;
        }
        toy_colsum<M>(sm->red, slot + lay.on_g, [&](int i) { return dh[i] * xh[i]; });
        toy_colsum<M>(sm->red, slot + lay.on_b, [&](int i) { return dh[i]; });
#pragma unroll
        for (int i = 0; i < M / 2; ++i) dh[i] *= sm->s.ong[toy_col(i)];
        toy_ln_bwd<M>(dh, xh, rstd);
        for (int l = a.L - 1; l >= 0; --l) {
            const float* ul = a.u_sv + (size_t)l * B * M;
            const float* hl = a.h_sv + (size_t)l * B * M;
            // ---- fc2 / LN2
#pragma unroll
            for (int i = 0; i < M / 2; ++i) acc[i] = ld(ul, i);
            toy_ln_stats<M>(acc, mean, rstd);
#pragma unroll
            for (int i = 0; i < M / 2; ++i) { const int r = (i >> 1) & 1; xh[i] = (acc[i] - mean[r]) * rstd[r]; }
            __syncthreads();
            toy_put<M>(sm->ta, [&](int i) { return dh[i]; });
            toy_put<M>(sm->tb, [&](int i) { const int c = toy_col(i); return toy_lrelu(xh[i] * sm->s.n2g[c] + sm->s.n2b[c]); });
            toy_sync_for_wgmma();
            toy_mm_wgrad<M>(acc, sm->ta, sm->tb, slot + lay.fc2);
            toy_mm_nn<M>(acc, sm->ta, sm->fc2);                     // d lrelu(LN2(u))
#pragma unroll
            for (int i = 0; i < M / 2; ++i) { const int c = toy_col(i); acc[i] *= toy_lrelu_grad(xh[i] * sm->s.n2g[c] + sm->s.n2b[c]); }
            toy_colsum<M>(sm->red, slot + lay.n2_g, [&](int i) { return acc[i] * xh[i]; });
            toy_colsum<M>(sm->red, slot + lay.n2_b, [&](int i) { return acc[i]; });
#pragma unroll
            for (int i = 0; i < M / 2; ++i) acc[i] *= sm->s.n2g[toy_col(i)];
            toy_ln_bwd<M>(acc, xh, rstd);                           // du
#pragma unroll
            for (int i = 0; i < M / 2; i += 2) {                    // dE = sum over the layers of du
                const int g = gr[(i >> 1) & 1];
                if (g >= B) continue;
                float2* p = reinterpret_cast<float2*>(a.dE + (size_t)g * M + toy_col(i));
                float2 v = l == a.L - 1 ? make_float2(0.f, 0.f) : *p;
                v.x += acc[i]; v.y += acc[i + 1];
                *p = v;
            }
            // ---- fc1 / LN1
#pragma unroll
            for (int i = 0; i < M / 2; ++i) xh[i] = ld(hl, i);
            toy_ln_stats<M>(xh, mean, rstd);
#pragma unroll
            for (int i = 0; i < M / 2; ++i) { const int r = (i >> 1) & 1; xh[i] = (xh[i] - mean[r]) * rstd[r]; }
            __syncthreads();
            toy_put<M>(sm->ta, [&](int i) { return acc[i]; });
            toy_put<M>(sm->tb, [&](int i) { const int c = toy_col(i); return toy_lrelu(xh[i] * sm->s.n1g[c] + sm->s.n1b[c]); });
            toy_sync_for_wgmma();
            toy_mm_wgrad<M>(acc, sm->ta, sm->tb, slot + lay.fc1);
            toy_mm_nn<M>(acc, sm->ta, sm->fc1);
#pragma unroll
            for (int i = 0; i < M / 2; ++i) { const int c = toy_col(i); acc[i] *= toy_lrelu_grad(xh[i] * sm->s.n1g[c] + sm->s.n1b[c]); }
            toy_colsum<M>(sm->red, slot + lay.n1_g, [&](int i) { return acc[i] * xh[i]; });
            toy_colsum<M>(sm->red, slot + lay.n1_b, [&](int i) { return acc[i]; });
#pragma unroll
            for (int i = 0; i < M / 2; ++i) acc[i] *= sm->s.n1g[toy_col(i)];
            toy_ln_bwd<M>(acc, xh, rstd);
#pragma unroll
            for (int i = 0; i < M / 2; ++i) dh[i] += acc[i];         // residual
        }
        // in_fc: dW_in(c, d) = sum_r dh(r, c) x(r, d);  dx(r, d) = sum_c dh(r, c) W_in(c, d)
        float x[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int d = 0; d < 4; ++d) x[r][d] = (gr[r] < B && d < D) ? a.x_sv[(size_t)gr[r] * D + d] : 0.f;
        for (int d = 0; d < D; ++d) {       // toy_colsum with the result scattered at stride D (in_fc.weight is [M][D])
            float s[M / 4];
#pragma unroll
            for (int j = 0; j < M / 8; ++j) {
                s[2 * j] = dh[4 * j] * x[0][d] + dh[4 * j + 2] * x[1][d];
                s[2 * j + 1] = dh[4 * j + 1] * x[0][d] + dh[4 * j + 3] * x[1][d];
            }
#pragma unroll
            for (int i = 0; i < M / 4; ++i) {
                s[i] += __shfl_xor_sync(0xffffffffu, s[i], 4); s[i] += __shfl_xor_sync(0xffffffffu, s[i], 8); s[i] += __shfl_xor_sync(0xffffffffu, s[i], 16);
            }
            if (lane < 4)
#pragma unroll
                for (int j = 0; j < M / 8; ++j) { sm->red[w * M + 8 * j + 2 * lane] = s[2 * j]; sm->red[w * M + 8 * j + 2 * lane + 1] = s[2 * j + 1]; }
            __syncthreads();
            if (threadIdx.x < M)
                slot[lay.in_w + (size_t)threadIdx.x * D + d] += ((sm->red[threadIdx.x] + sm->red[M + threadIdx.x]) + sm->red[2 * M + threadIdx.x]) + sm->red[3 * M + threadIdx.x];
            __syncthreads();
        }
        if (a.dx) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int i = 0; i < M / 2; ++i)
                    if (((i >> 1) & 1) == r)
#pragma unroll
                        for (int d = 0; d < 4; ++d) v[d] += dh[i] * sm->s.in_w[toy_col(i)][d];
#pragma unroll
                for (int d = 0; d < 4; ++d) v[d] = quad_sum(v[d]);
                if (gr[r] < B && q < D) a.dx[(size_t)gr[r] * D + q] = q == 0 ? v[0] : q == 1 ? v[1] : q == 2 ? v[2] : v[3];
            }
        }
    }
}

// dE -> partials of enc (weight, bias) and t_proj (weight, bias); the timestep path is recomputed from t
template <int M>
__global__ void __launch_bounds__(TOY_THREADS) toy_temb_bwd_kernel(const ToyArgs a) {
    pdl_entry();
    extern __shared__ uint8_t smem_raw[];
    auto* sm = reinterpret_cast<ToyTembSmem<M>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    toy_stage_w(sm->tp, a.w.t_proj_weight, M, M);
    toy_stage_w(sm->enc, a.w.enc_weight, M, M);
    const ToyLayout lay(M, a.D, a.L);
    float* slot = a.part + (size_t)blockIdx.x * lay.Pp;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int B = a.B;
    float pre[M / 2], d[M / 2];
    for (int tile = blockIdx.x; tile < toy_tiles(B); tile += gridDim.x) {
        const int row0 = tile * 64, g0 = row0 + 16 * w + (lane >> 2);
        toy_temb_tile<M>(pre, sm, a, row0, B);                      // ta = emb, tb = e
#pragma unroll
        for (int i = 0; i < M / 2; ++i) { const int g = g0 + 8 * ((i >> 1) & 1); d[i] = g < B ? a.dE[(size_t)g * M + toy_col(i)] : 0.f; }
        toy_put<M>(sm->td, [&](int i) { return d[i]; });
        toy_sync_for_wgmma();
        toy_colsum<M>(sm->red, slot + lay.enc_b, [&](int i) { return d[i]; });
        toy_mm_wgrad<M>(d, sm->td, sm->tb, slot + lay.enc_w);
        toy_mm_nn<M>(d, sm->td, sm->enc);                           // de
#pragma unroll
        for (int i = 0; i < M / 2; ++i) d[i] *= toy_lrelu_grad(pre[i]);
        toy_colsum<M>(sm->red, slot + lay.tp_b, [&](int i) { return d[i]; });
        toy_put<M>(sm->td, [&](int i) { return d[i]; });           // the wgmmas that read td have completed (colsum's barriers)
        toy_sync_for_wgmma();
        toy_mm_wgrad<M>(d, sm->td, sm->ta, slot + lay.tp_w);
    }
}

// flat[i] = sum over the slots in slot order
__global__ void toy_reduce_kernel(const float* __restrict__ part, int slots, long long P, long long Pp, float* __restrict__ flat) {
    pdl_entry();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float s = 0.f;
    for (int k = 0; k < slots; ++k) s += part[(size_t)k * Pp + i];
    flat[i] = s;
}

// ------------------------------------------------------------------------------------------------ sampler chain
// coef [S][6] = {sqrt_recip_ab, sqrt_recip_m1_ab, c1, c2, sigma, t>0} (fp32 as the mirror's p_sample_step sees them);
// z [S][B][D]: z[k] is the noise of the k-th step (t = S-1-k).  x_0 prediction is NOT clipped (toy/diffusion.py:33).
template <int M>
__global__ void __launch_bounds__(TOY_THREADS) toy_sample_kernel(const ToyArgs a) {
    pdl_entry();
    extern __shared__ uint8_t smem_raw[];
    auto* sm = reinterpret_cast<ToyFwdSmem<M>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    toy_stage_w(sm->fc1, a.w.fc1_weight, M, M);
    toy_stage_w(sm->fc2, a.w.fc2_weight, M, M);
    toy_stage_small<M>(&sm->s, a);
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, q = lane & 3;
    const int D = a.D, B = a.B;
    float* X = const_cast<float*>(a.x);
    float h[M / 2], u[M / 2];
    for (int tile = blockIdx.x; tile < toy_tiles(B); tile += gridDim.x) {
        const int g0 = tile * 64 + 16 * w + (lane >> 2);
        const int gr[2] = {g0, g0 + 8};
        float x[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int d = 0; d < 4; ++d) x[r][d] = (gr[r] < B && d < D) ? X[(size_t)gr[r] * D + d] : 0.f;
        for (int k = 0; k < a.S; ++k) {
            const int ti = a.S - 1 - k;
            const float* Et = a.E + (size_t)ti * M;
            toy_in_fc<M>(h, x, &sm->s);
            for (int l = 0; l < a.L; ++l) toy_layer<M>(h, u, sm, [&](int i) { return __ldg(Et + toy_col(i)); });
            float eps[2][4];
            toy_head<M>(h, &sm->s, eps);
            const float* cf = a.coef + (size_t)ti * 6;
            const float ra = cf[0], rb = cf[1], c1 = cf[2], c2 = cf[3], sg = __fmul_rn(cf[5], cf[4]);
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int d = 0; d < 4; ++d) {
                    const float z = (gr[r] < B && d < D) ? a.z[((size_t)k * B + gr[r]) * D + d] : 0.f;
                    const float x0 = __fsub_rn(__fmul_rn(ra, x[r][d]), __fmul_rn(rb, eps[r][d]));
                    const float mean = __fadd_rn(__fmul_rn(c1, x0), __fmul_rn(c2, x[r][d]));
                    x[r][d] = __fadd_rn(mean, __fmul_rn(sg, z));
                }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r)
            if (gr[r] < B && q < D) X[(size_t)gr[r] * D + q] = q == 0 ? x[r][0] : q == 1 ? x[r][1] : q == 2 ? x[r][2] : x[r][3];
    }
}

// ------------------------------------------------------------------------------------------------ host side
inline size_t toy_align(size_t b) { return (b + 255) & ~size_t(255); }
inline int toy_grid(int rows, int cap) { const int t = (rows + 63) / 64; return t < cap ? t : cap; }

struct ToyWs { size_t E, h, u, x, out, dE, part, total; };
// training = 0: E [rows][M] only.  training = 1: + the saves, dE and one partial slot per backward CTA
inline ToyWs toy_ws_layout(int M, int D, int L, long long rows, int training) {
    ToyWs w{};
    size_t o = 0;
    w.E = o; o += toy_align((size_t)rows * M * 4);
    if (training) {
        const ToyLayout lay(M, D, L);
        w.h = o; o += toy_align((size_t)(L + 1) * rows * M * 4);
        w.u = o; o += toy_align((size_t)L * rows * M * 4);
        w.x = o; o += toy_align((size_t)rows * D * 4);
        w.out = o; o += toy_align((size_t)rows * D * 4);
        w.dE = o; o += toy_align((size_t)rows * M * 4);
        w.part = o; o += toy_align((size_t)toy_grid((int)rows, TOY_BWD_CTAS) * lay.Pp * 4);
    }
    w.total = o;
    return w;
}

template <int M> inline size_t toy_smem_fwd() { return sizeof(ToyFwdSmem<M>) + 1024; }
template <int M> inline size_t toy_smem_bwd() { return sizeof(ToyBwdSmem<M>) + 1024; }
template <int M> inline size_t toy_smem_temb() { return sizeof(ToyTembSmem<M>) + 1024; }

template <typename K>
inline cudaError_t toy_launch(K kern, int grid, size_t shm, cudaStream_t st, const ToyArgs& a) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
    if (e != cudaSuccess) return e;
    e = launch_k(kern, dim3(grid), dim3(TOY_THREADS), shm, st, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <int M>
inline cudaError_t toy_temb_launch(const ToyArgs& a, int rows, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(toy_temb_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)toy_smem_temb<M>());
    if (e != cudaSuccess) return e;
    e = launch_k(toy_temb_kernel<M>, dim3(toy_grid(rows, TOY_FWD_CTAS)), dim3(TOY_THREADS), toy_smem_temb<M>(), st, a, rows);
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <int M>
inline cudaError_t toy_forward_launch(const ToyArgs& a, cudaStream_t st) {
    cudaError_t e = toy_temb_launch<M>(a, a.B, st);
    return e != cudaSuccess ? e : toy_launch(toy_fwd_kernel<M>, toy_grid(a.B, TOY_FWD_CTAS), toy_smem_fwd<M>(), st, a);
}

template <int M>
inline cudaError_t toy_backward_launch(const ToyArgs& a, float* grad, cudaStream_t st) {
    const ToyLayout lay(M, a.D, a.L);
    const int grid = toy_grid(a.B, TOY_BWD_CTAS);
    cudaError_t e = cudaMemsetAsync(a.part, 0, (size_t)grid * lay.Pp * 4, st);
    if (e == cudaSuccess) e = toy_launch(toy_bwd_kernel<M>, grid, toy_smem_bwd<M>(), st, a);
    if (e == cudaSuccess) e = toy_launch(toy_temb_bwd_kernel<M>, grid, toy_smem_temb<M>(), st, a);
    if (e != cudaSuccess) return e;
    e = launch_k(toy_reduce_kernel, dim3((unsigned)((lay.P + 255) / 256)), dim3(256), 0, st, (const float*)a.part, grid, lay.P, lay.Pp, grad);
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <int M>
inline cudaError_t toy_sample_launch(const ToyArgs& a, cudaStream_t st) {
    cudaError_t e = toy_temb_launch<M>(a, a.S, st);
    return e != cudaSuccess ? e : toy_launch(toy_sample_kernel<M>, toy_grid(a.B, TOY_FWD_CTAS), toy_smem_fwd<M>(), st, a);
}

}  // namespace ddpm
