// FID Inception-v3 forward (ddpm_torch/metrics/inception.py): 94 BasicConv2d layers (bias-free conv, eval BatchNorm eps = 1e-3,
// ReLU), the max / average pools between them and the global average at the end, on NHWC fp32 activations.
//
// Convolution.  One kernel, inc_conv_tf32_kernel: an implicit GEMM on the sm_90a tensor cores with TF32 operands (wgmma
// m64nNk8 .tf32), M = N Ho Wo output pixels, N = Cout, K = kh kw Cin4 (Cin4 = Cin rounded up to 4; k = (ky kw + kx) Cin4 + ci).
// Every thread of the CTA gathers: 16-byte cp.async chunks of the im2col rows (zero-filled outside the image and past K) and of
// the packed weight rows land in a 128-byte-swizzled, K-major stage ring; the thread rounds its own activation chunks to TF32
// (cvt.rna) once they have landed, so both operands reach the tensor core already rounded to nearest (the weights are rounded
// when they are packed).  Two consumer warpgroups each own 64 rows of the 128-row tile and issue the wgmmas of one 32-wide K
// block per stage.  The epilogue adds the folded BatchNorm bias, applies ReLU and stores fp32 straight into channels
// [c_off, c_off + Cout) of an NHWC tensor with C_total channels, which is how every torch.cat of the blocks is made free.
// No split-K, no atomics: an output element is one CTA's fixed-order sum over K, so an image's features do not depend on the
// batch it arrives in or on the call.
//
// Everything else is plain SIMT: the input kernel (bilinear resize to 299 x 299 as F.interpolate(align_corners=False) computes it,
// 2x - 1, NCHW -> NHWC with 4 channels), the 3 x 3 pools, the global average, the NHWC -> NCHW copy of a block output and, on
// request, the gather of sFID's spatial features (channels 0..6 of Mixed_6d's output) while that output is still in its buffer.
#pragma once
#include <climits>
#include <string>
#include <vector>
#include "ptx.cuh"

namespace ddpm {

constexpr int INC_BM = 128;                    // output pixels per CTA (two warpgroups x 64)
constexpr int INC_BK = 32;                     // K per stage: one 128-byte swizzled row of fp32
constexpr int INC_STAGES = 6;                  // stage ring
constexpr int INC_PREFETCH = INC_STAGES - 2;   // K blocks in flight; the 2 spare stages cover the wgmma group still reading
constexpr int INC_THREADS = 256;
constexpr int INC_COUT_PAD = 128;              // packed weights: Cout rounded up to this, K rounded up to INC_BK
constexpr double INC_BN_EPS = 1e-3;
constexpr int INC_NUM_CONVS = 94;
constexpr int INC_FIELDS = 5;                  // conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var

// ------------------------------------------------------------------------------------------------ wgmma .tf32 (K-major A and B)
__device__ __forceinline__ void wgmma_tf32_m64n64(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_m64n128(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(1));
}
template <int BN> __device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 64) wgmma_tf32_m64n64(d, da, db); else wgmma_tf32_m64n128(d, da, db);
}

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint32_t tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// ------------------------------------------------------------------------------------------------ convolution
struct IncConvArgs {
    const float* x; int H, W, Cin4;            // NHWC input, pitch Cin4 (a multiple of 4)
    int Ho, Wo, kw, stride, ph, pw;
    int K, KT;                                 // K = kh kw Cin4, KT = ceil(K / INC_BK)
    const float* w; const float* bias;         // packed: w [Cout_pad][KT * INC_BK] (TF32 values), bias [Cout_pad]
    float* out; int Cout, c_off, C_total;
    int M, n_tiles;                            // M = N Ho Wo; CTAs run the Cout tiles of one pixel tile back to back
};

template <int BN>
__host__ __device__ constexpr int inc_stage_bytes() { return INC_BM * INC_BK * 4 + BN * INC_BK * 4; }
template <int BN>
__host__ __device__ constexpr int inc_smem_bytes() { return INC_STAGES * inc_stage_bytes<BN>() + 1024; }

// Chunk c (16 bytes) of row r of a 128-byte-swizzled K-major tile lives at r * 128 + ((c ^ (r & 7)) << 4).
__device__ __forceinline__ uint32_t inc_swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// The GEMM body shared by the convolutions and the Inception Score's logits (inception_score.cuh).  BN_RELU: the convolutions'
// epilogue (folded BatchNorm bias, then ReLU); without it the raw fp32 accumulators are stored.
template <int BN, bool BN_RELU>
__device__ __forceinline__ void inc_conv_tf32_body(const IncConvArgs& a) {
    extern __shared__ uint8_t inc_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(inc_smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int STAGE = inc_stage_bytes<BN>();
    constexpr int A_BYTES = INC_BM * INC_BK * 4;
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;
    const int m_tile = blockIdx.x / a.n_tiles, n_tile = blockIdx.x - m_tile * a.n_tiles;
    const int m0 = m_tile * INC_BM, n0 = n_tile * BN;
    pdl_entry();

    // producer role: chunk c of rows (tid >> 3) + 32 i of the A tile and (tid >> 3) + 32 j of the B tile
    const int c = tid & 7, r0 = tid >> 3;
    int pix[4], iy0[4], ix0[4];
    const int HoWo = a.Ho * a.Wo;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + r0 + 32 * i;
        if (m < a.M) {
            const int n = m / HoWo, rem = m - n * HoWo, oy = rem / a.Wo, ox = rem - oy * a.Wo;
            pix[i] = n * a.H * a.W; iy0[i] = oy * a.stride - a.ph; ix0[i] = ox * a.stride - a.pw;
        } else {
            pix[i] = 0; iy0[i] = INT_MIN / 2; ix0[i] = 0;          // never inside the image
        }
    }
    const long long ldw = (long long)a.KT * INC_BK;
    auto load_stage = [&](int kt, int slot) {
        uint8_t* sa = smem + slot * STAGE;
        uint8_t* sb = sa + A_BYTES;
        const int k = kt * INC_BK + 4 * c;
        const bool kv = k < a.K;
        const int tap = k / a.Cin4, ci = k - tap * a.Cin4, ky = tap / a.kw, kx = tap - ky * a.kw;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = r0 + 32 * i, iy = iy0[i] + ky, ix = ix0[i] + kx;
            const bool v = kv && (unsigned)iy < (unsigned)a.H && (unsigned)ix < (unsigned)a.W;
            const float* src = v ? a.x + (long long)(pix[i] + iy * a.W + ix) * a.Cin4 + ci : a.x;
            cp_async16_zfill(sa + inc_swz(r, c), src, v);
        }
#pragma unroll
        for (int j = 0; j < BN / 32; ++j) {
            const int r = r0 + 32 * j;
            cp_async16_zfill(sb + inc_swz(r, c), a.w + (long long)(n0 + r) * ldw + kt * INC_BK + 4 * c, true);
        }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < INC_PREFETCH; ++s) {
        if (s < a.KT) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < a.KT; ++kt) {
        const int slot = kt % INC_STAGES;
        cp_async_wait<INC_PREFETCH - 1>();                       // this thread's chunks of K block kt have landed
        uint8_t* sa = smem + slot * STAGE;
#pragma unroll
        for (int i = 0; i < 4; ++i) {                            // round them to TF32 in place
            uint8_t* p = sa + inc_swz(r0 + 32 * i, c);
            uint32_t u0, u1, u2, u3;
            ld_shared_v4(p, u0, u1, u2, u3);
            st_shared_v4(p, tf32_rna(__uint_as_float(u0)), tf32_rna(__uint_as_float(u1)), tf32_rna(__uint_as_float(u2)),
                         tf32_rna(__uint_as_float(u3)));
        }
        fence_proxy_async_smem();
        // after this barrier every warpgroup has also retired its wgmmas of K block kt - 2 (wgmma_wait<1> below), so that block's
        // stage is free for the prefetch of K block kt + INC_PREFETCH
        __syncthreads();
        if (kt + INC_PREFETCH < a.KT) load_stage(kt + INC_PREFETCH, (kt + INC_PREFETCH) % INC_STAGES);
        cp_async_commit();
        const uint32_t a_base = smem_u32(sa) + wg * (64 * 128), b_base = smem_u32(sa + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < INC_BK / 8; ++kk)
            wgmma_tf32<BN>(acc, wg_smem_desc(a_base + 32 * kk, 16, 1024), wg_smem_desc(b_base + 32 * kk, 16, 1024));
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    cp_async_wait<0>();

    const int w = wt >> 5, l = wt & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + wg * 64 + 16 * w + (l >> 2) + 8 * h;
        if (m >= a.M) continue;
        float* orow = a.out + (long long)m * a.C_total + a.c_off;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = n0 + 8 * j + 2 * (l & 3);
            if (col < a.Cout) {                                  // Cout is even: col + 1 < Cout too
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if constexpr (BN_RELU) {
                    v0 += __ldg(a.bias + col); v1 += __ldg(a.bias + col + 1);
                    v0 = v0 < 0.f ? 0.f : v0; v1 = v1 < 0.f ? 0.f : v1;
                }
                *reinterpret_cast<float2*>(orow + col) = make_float2(v0, v1);
            }
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(INC_THREADS, 1) inc_conv_tf32_kernel(const IncConvArgs a) { inc_conv_tf32_body<BN, true>(a); }

// BatchNorm folded into the conv, in fp64, rounded once to fp32 and then to TF32 (the value the tensor core multiplies):
// w' = w gamma / sqrt(var + eps) laid out [Cout_pad][Kp] with k = (ky kw + kx) Cin4 + ci, zero outside the layer;
// b' = beta - mean gamma / sqrt(var + eps), zero past Cout.  With `split` (Cin4 = 12) the three 4-channel groups of a tap hold
// w_hi = tf32(w'), w_hi and w_lo = tf32(w' - w_hi): against the split image that is x_hi w_hi + x_lo w_hi + x_hi w_lo, the
// 3xTF32 product, accurate to about 2^-21 instead of 2^-10.
__global__ void k_inc_fold(const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
                           const float* __restrict__ mean, const float* __restrict__ var, int Cin, int Cin4, int kh, int kw, int Cout,
                           int Cout_pad, int Kp, float* __restrict__ wp, float* __restrict__ bp, int split) {
    pdl_entry();
    const long long nw = (long long)Cout_pad * Kp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nw + Cout_pad; i += (long long)gridDim.x * blockDim.x) {
        if (i < nw) {
            const int co = (int)(i / Kp), k = (int)(i - (long long)co * Kp);
            const int tap = k / Cin4, cs = k - tap * Cin4, part = split ? cs >> 2 : 0, ci = split ? cs & 3 : cs;
            float v = 0.f;
            if (co < Cout && tap < kh * kw && ci < Cin) {
                const int ky = tap / kw, kx = tap - ky * kw;
                const double s = (double)w[(((long long)co * Cin + ci) * kh + ky) * kw + kx] * (double)gamma[co] /
                                 sqrt((double)var[co] + INC_BN_EPS);
                const float f = __double2float_rn(s), hi = __uint_as_float(tf32_rna(f));
                v = part < 2 ? hi : __uint_as_float(tf32_rna(f - hi));     // split: [w_hi | w_hi | w_lo] against [x_hi | x_lo | x_hi]
            }
            wp[i] = v;
        } else {
            const int co = (int)(i - nw);
            bp[co] = co < Cout ? __double2float_rn((double)beta[co] - (double)mean[co] * (double)gamma[co] /
                                                   sqrt((double)var[co] + INC_BN_EPS))
                               : 0.f;
        }
    }
}

// ------------------------------------------------------------------------------------------------ SIMT kernels
// F.interpolate(size=(299, 299), mode="bilinear", align_corners=False) of CUDA upsample_bilinear2d, then 2x - 1; NCHW [N][3][H][W]
// in, NHWC [N][Ho][Wo][12] out: {x_hi, 0, x_lo, 0, x_hi, 0} with x_hi = tf32(x) (3 channels) and x_lo = x - x_hi (exact).  The
// first conv reads the image at 3xTF32 accuracy this way: its error would otherwise be the largest single TF32 rounding of the
// input, which cuDNN's fp32 kernels for a 3-channel conv do not make.
__global__ void k_inc_input(const float* __restrict__ x, int N, int H, int W, int Ho, int Wo, int resize, int normalize,
                            float* __restrict__ out) {
    pdl_entry();
    const long long total = (long long)N * Ho * Wo;
    const float rh = (float)H / Ho, rw = (float)W / Wo;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(p / ((long long)Ho * Wo)), rem = (int)(p - (long long)n * Ho * Wo), oy = rem / Wo, ox = rem - oy * Wo;
        const float* img = x + (long long)n * 3 * H * W;
        float v[3];
        if (resize) {
            float sy = rh * (oy + 0.5f) - 0.5f, sx = rw * (ox + 0.5f) - 0.5f;
            sy = sy < 0.f ? 0.f : sy; sx = sx < 0.f ? 0.f : sx;
            const int y1 = (int)sy, x1 = (int)sx;
            const int y1p = y1 < H - 1 ? 1 : 0, x1p = x1 < W - 1 ? 1 : 0;
            const float l1y = sy - y1, l0y = 1.f - l1y, l1x = sx - x1, l0x = 1.f - l1x;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float* q = img + (long long)ch * H * W + (long long)y1 * W + x1;
                v[ch] = l0y * (l0x * q[0] + l1x * q[x1p]) + l1y * (l0x * q[y1p * W] + l1x * q[y1p * W + x1p]);
            }
        } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) v[ch] = img[(long long)ch * H * W + (long long)oy * W + ox];
        }
        if (normalize) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) v[ch] = __fsub_rn(__fmul_rn(2.f, v[ch]), 1.f);
        }
        float hi[3], lo[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) { hi[ch] = __uint_as_float(tf32_rna(v[ch])); lo[ch] = v[ch] - hi[ch]; }
        float4* o = reinterpret_cast<float4*>(out) + 3 * p;
        o[0] = make_float4(hi[0], hi[1], hi[2], 0.f);
        o[1] = make_float4(lo[0], lo[1], lo[2], 0.f);
        o[2] = make_float4(hi[0], hi[1], hi[2], 0.f);
    }
}

enum IncPool { INC_MAX3_S2 = 0, INC_AVG3_S1 = 1, INC_MAX3_S1 = 2 };
inline void inc_pool_dims(int kind, int H, int W, int& Ho, int& Wo) {
    if (kind == INC_MAX3_S2) { Ho = H >= 3 ? (H - 3) / 2 + 1 : 0; Wo = W >= 3 ? (W - 3) / 2 + 1 : 0; }
    else { Ho = H; Wo = W; }
}

// 3 x 3 pools on NHWC [N][H][W][C] into channels [c_off, c_off + C) of [N][Ho][Wo][C_total]: max stride 2 without padding
// (nn.MaxPool2d(3, 2)), average stride 1 padding 1 over the window's in-image taps only (count_include_pad=False), max stride 1
// padding 1.  Max keeps a NaN as torch does; the average sums in torch's order (rows, then columns) and divides by the count.
__global__ void k_inc_pool(const float* __restrict__ x, int N, int H, int W, int C, int kind, int Ho, int Wo, float* __restrict__ out,
                           int c_off, int C_total) {
    pdl_entry();
    const long long total = (long long)N * Ho * Wo * C;
    const int stride = kind == INC_MAX3_S2 ? 2 : 1, pad = kind == INC_MAX3_S2 ? 0 : 1;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / C;
        const int ch = (int)(i - p * C);
        const int n = (int)(p / ((long long)Ho * Wo)), rem = (int)(p - (long long)n * Ho * Wo), oy = rem / Wo, ox = rem - oy * Wo;
        const int ys = oy * stride - pad, xs = ox * stride - pad;
        const int y0 = ys < 0 ? 0 : ys, y1 = ys + 3 < H ? ys + 3 : H, x0 = xs < 0 ? 0 : xs, x1 = xs + 3 < W ? xs + 3 : W;
        const float* img = x + (long long)n * H * W * C + ch;
        float r;
        if (kind == INC_AVG3_S1) {
            float s = 0.f;
            for (int y = y0; y < y1; ++y)
                for (int xx = x0; xx < x1; ++xx) s += img[((long long)y * W + xx) * C];
            r = s / (float)((y1 - y0) * (x1 - x0));
        } else {
            r = -INFINITY;
            for (int y = y0; y < y1; ++y)
                for (int xx = x0; xx < x1; ++xx) {
                    const float v = img[((long long)y * W + xx) * C];
                    if (v > r || isnan(v)) r = v;
                }
        }
        out[p * C_total + c_off + ch] = r;
    }
}

// Global average of NHWC [N][HW][C] -> rows out[n * ld + c], summed in pixel order.
__global__ void k_inc_gap(const float* __restrict__ x, int N, int HW, int C, float* __restrict__ out, int ld) {
    pdl_entry();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)N * C; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i / C), ch = (int)(i - (long long)n * C);
        const float* p = x + (long long)n * HW * C + ch;
        float s = 0.f;
        for (int q = 0; q < HW; ++q) s += p[(long long)q * C];
        out[(long long)n * ld + ch] = s / (float)HW;
    }
}

// NHWC [N][HW][C] -> NCHW [N][C][HW] (a block output as the torch module returns it)
__global__ void k_inc_nchw(const float* __restrict__ x, int N, int HW, int C, float* __restrict__ out) {
    pdl_entry();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)N * C * HW; i += (long long)gridDim.x * blockDim.x) {
        const long long n = i / ((long long)C * HW);
        const long long rem = i - n * C * HW;
        const int ch = (int)(rem / HW), q = (int)(rem - (long long)ch * HW);
        out[i] = x[(n * HW + q) * C + ch];
    }
}

// sFID's spatial features (Nash et al., 2021, as the guided-diffusion evaluator reads mixed_6/conv:0[..., :7]): channels
// [0, INC_SPATIAL_C) of NHWC [N][HW][C] -> rows out[n][p * INC_SPATIAL_C + c], p = h W + w, i.e. TensorFlow's NHWC flatten.  Pixel
// q = n HW + p of the input lands at q * INC_SPATIAL_C + c of the output, so the output is written in order, one float per thread.
constexpr int INC_SPATIAL_C = 7;
__global__ void k_sfid_gather(const float* __restrict__ x, long long pixels, int C, float* __restrict__ out) {
    pdl_entry();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < pixels * INC_SPATIAL_C; i += (long long)gridDim.x * blockDim.x) {
        const long long q = i / INC_SPATIAL_C;
        out[i] = x[q * C + (i - q * INC_SPATIAL_C)];
    }
}

// ------------------------------------------------------------------------------------------------ host side: the layer table
// split: the network's first conv reads the input kernel's 12-channel split image (see k_inc_input) and is packed to match
struct IncConv { int cin, cout, kh, kw, stride, ph, pw; std::string name; bool split = false; };

inline int inc_cin4(const IncConv& c) { return c.split ? 12 : (c.cin + 3) / 4 * 4; }
inline int inc_kp(const IncConv& c) { return (c.kh * c.kw * inc_cin4(c) + INC_BK - 1) / INC_BK * INC_BK; }
inline int inc_cout_pad(int cout) { return (cout + INC_COUT_PAD - 1) / INC_COUT_PAD * INC_COUT_PAD; }

// The 94 BasicConv2d layers of torchvision's Inception3 as fid_inception_v3 assembles it, in state_dict order, which is also
// the order the forward runs them in.
inline const std::vector<IncConv>& inc_convs() {
    static const std::vector<IncConv> v = [] {
        std::vector<IncConv> t;
        auto add = [&](const std::string& n, int ci, int co, int kh, int kw, int s = 1, int ph = 0, int pw = 0) {
            t.push_back({ci, co, kh, kw, s, ph, pw, n});
        };
        add("Conv2d_1a_3x3", 3, 32, 3, 3, 2);
        t.back().split = true;
        add("Conv2d_2a_3x3", 32, 32, 3, 3);
        add("Conv2d_2b_3x3", 32, 64, 3, 3, 1, 1, 1);
        add("Conv2d_3b_1x1", 64, 80, 1, 1);
        add("Conv2d_4a_3x3", 80, 192, 3, 3);
        const struct { const char* n; int cin, pf; } A[] = {{"Mixed_5b", 192, 32}, {"Mixed_5c", 256, 64}, {"Mixed_5d", 288, 64}};
        for (auto& b : A) {
            const std::string p = std::string(b.n) + ".";
            add(p + "branch1x1", b.cin, 64, 1, 1);
            add(p + "branch5x5_1", b.cin, 48, 1, 1);
            add(p + "branch5x5_2", 48, 64, 5, 5, 1, 2, 2);
            add(p + "branch3x3dbl_1", b.cin, 64, 1, 1);
            add(p + "branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1);
            add(p + "branch3x3dbl_3", 96, 96, 3, 3, 1, 1, 1);
            add(p + "branch_pool", b.cin, b.pf, 1, 1);
        }
        add("Mixed_6a.branch3x3", 288, 384, 3, 3, 2);
        add("Mixed_6a.branch3x3dbl_1", 288, 64, 1, 1);
        add("Mixed_6a.branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1);
        add("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 3, 2);
        const struct { const char* n; int c7; } Cb[] = {{"Mixed_6b", 128}, {"Mixed_6c", 160}, {"Mixed_6d", 160}, {"Mixed_6e", 192}};
        for (auto& b : Cb) {
            const std::string p = std::string(b.n) + ".";
            const int c7 = b.c7;
            add(p + "branch1x1", 768, 192, 1, 1);
            add(p + "branch7x7_1", 768, c7, 1, 1);
            add(p + "branch7x7_2", c7, c7, 1, 7, 1, 0, 3);
            add(p + "branch7x7_3", c7, 192, 7, 1, 1, 3, 0);
            add(p + "branch7x7dbl_1", 768, c7, 1, 1);
            add(p + "branch7x7dbl_2", c7, c7, 7, 1, 1, 3, 0);
            add(p + "branch7x7dbl_3", c7, c7, 1, 7, 1, 0, 3);
            add(p + "branch7x7dbl_4", c7, c7, 7, 1, 1, 3, 0);
            add(p + "branch7x7dbl_5", c7, 192, 1, 7, 1, 0, 3);
            add(p + "branch_pool", 768, 192, 1, 1);
        }
        add("Mixed_7a.branch3x3_1", 768, 192, 1, 1);
        add("Mixed_7a.branch3x3_2", 192, 320, 3, 3, 2);
        add("Mixed_7a.branch7x7x3_1", 768, 192, 1, 1);
        add("Mixed_7a.branch7x7x3_2", 192, 192, 1, 7, 1, 0, 3);
        add("Mixed_7a.branch7x7x3_3", 192, 192, 7, 1, 1, 3, 0);
        add("Mixed_7a.branch7x7x3_4", 192, 192, 3, 3, 2);
        const struct { const char* n; int cin; } E[] = {{"Mixed_7b", 1280}, {"Mixed_7c", 2048}};
        for (auto& b : E) {
            const std::string p = std::string(b.n) + ".";
            add(p + "branch1x1", b.cin, 320, 1, 1);
            add(p + "branch3x3_1", b.cin, 384, 1, 1);
            add(p + "branch3x3_2a", 384, 384, 1, 3, 1, 0, 1);
            add(p + "branch3x3_2b", 384, 384, 3, 1, 1, 1, 0);
            add(p + "branch3x3dbl_1", b.cin, 448, 1, 1);
            add(p + "branch3x3dbl_2", 448, 384, 3, 3, 1, 1, 1);
            add(p + "branch3x3dbl_3a", 384, 384, 1, 3, 1, 0, 1);
            add(p + "branch3x3dbl_3b", 384, 384, 3, 1, 1, 1, 0);
            add(p + "branch_pool", b.cin, 192, 1, 1);
        }
        return t;
    }();
    return v;
}

// raw parameter inventory (torchvision state_dict order, num_batches_tracked and fc.* left out): 5 tensors per conv
struct IncParam { std::string name; int ndim; int dims[4]; long long offset; };
inline const std::vector<IncParam>& inc_params() {
    static const std::vector<IncParam> v = [] {
        std::vector<IncParam> t;
        long long off = 0;
        static const char* field[INC_FIELDS] = {"conv.weight", "bn.weight", "bn.bias", "bn.running_mean", "bn.running_var"};
        for (const IncConv& c : inc_convs())
            for (int f = 0; f < INC_FIELDS; ++f) {
                IncParam p{c.name + "." + field[f], f == 0 ? 4 : 1, {c.cout, f == 0 ? c.cin : 0, f == 0 ? c.kh : 0, f == 0 ? c.kw : 0}, off};
                off += f == 0 ? (long long)c.cout * c.cin * c.kh * c.kw : c.cout;
                t.push_back(p);
            }
        return t;
    }();
    return v;
}

// packed layout: per conv, w [Cout_pad][Kp] then bias [Cout_pad], each at a 64-float (256-byte) boundary
inline long long inc_al64(long long n) { return (n + 63) / 64 * 64; }
inline const std::vector<long long>& inc_packed_offsets() {     // 2 per conv (w, bias), then the total
    static const std::vector<long long> v = [] {
        std::vector<long long> t;
        long long off = 0;
        for (const IncConv& c : inc_convs()) {
            t.push_back(off); off += inc_al64((long long)inc_cout_pad(c.cout) * inc_kp(c));
            t.push_back(off); off += inc_al64(inc_cout_pad(c.cout));
        }
        t.push_back(off);
        return t;
    }();
    return v;
}

inline int inc_grid(long long work, int per_block = 256) {
    const long long g = (work + per_block - 1) / per_block;
    return (int)(g < 1 ? 1 : g > 65536LL * 8 ? 65536LL * 8 : g);
}

inline cudaError_t inc_fold_launch(const IncConv& c, const float* w, const float* gamma, const float* beta, const float* mean,
                                   const float* var, float* wp, float* bp, cudaStream_t st) {
    const int cp = inc_cout_pad(c.cout), kp = inc_kp(c);
    return launch_k(k_inc_fold, dim3(inc_grid((long long)cp * kp + cp)), dim3(256), 0, st, w, gamma, beta, mean, var, c.cin,
                    inc_cin4(c), c.kh, c.kw, c.cout, cp, kp, wp, bp, (int)c.split);
}

inline int inc_conv_out(int H, int k, int s, int p) { return H + 2 * p >= k ? (H + 2 * p - k) / s + 1 : 0; }

template <int BN>
inline cudaError_t inc_conv_launch_bn(IncConvArgs a, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        const cudaError_t e = cudaFuncSetAttribute(inc_conv_tf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, inc_smem_bytes<BN>());
        if (e != cudaSuccess) return e;
        attr = true;
    }
    a.n_tiles = (a.Cout + BN - 1) / BN;
    const long long grid = (long long)((a.M + INC_BM - 1) / INC_BM) * a.n_tiles;
    return launch_k(inc_conv_tf32_kernel<BN>, dim3((unsigned)grid), dim3(INC_THREADS), inc_smem_bytes<BN>(), st, a);
}

// one conv of the table: x NHWC [N][H][W][Cin4], packed w / bias, out channels [c_off, c_off + Cout) of [N][Ho][Wo][C_total]
inline cudaError_t inc_conv_launch(const IncConv& c, const float* x, int N, int H, int W, const float* wp, const float* bp,
                                   float* out, int c_off, int C_total, cudaStream_t st) {
    IncConvArgs a;
    a.x = x; a.H = H; a.W = W; a.Cin4 = inc_cin4(c);
    a.Ho = inc_conv_out(H, c.kh, c.stride, c.ph); a.Wo = inc_conv_out(W, c.kw, c.stride, c.pw);
    a.kw = c.kw; a.stride = c.stride; a.ph = c.ph; a.pw = c.pw;
    a.K = c.kh * c.kw * a.Cin4; a.KT = inc_kp(c) / INC_BK;
    a.w = wp; a.bias = bp; a.out = out; a.Cout = c.cout; a.c_off = c_off; a.C_total = C_total;
    a.M = N * a.Ho * a.Wo; a.n_tiles = 0;
    return c.cout <= 64 ? inc_conv_launch_bn<64>(a, st) : inc_conv_launch_bn<128>(a, st);
}

inline cudaError_t inc_pool_launch(int kind, const float* x, int N, int H, int W, int C, float* out, int c_off, int C_total,
                                   cudaStream_t st) {
    int Ho, Wo;
    inc_pool_dims(kind, H, W, Ho, Wo);
    return launch_k(k_inc_pool, dim3(inc_grid((long long)N * Ho * Wo * C)), dim3(256), 0, st, x, N, H, W, C, kind, Ho, Wo, out, c_off,
                    C_total);
}

inline cudaError_t inc_input_launch(const float* x, int N, int H, int W, int resize, int normalize, float* out, cudaStream_t st) {
    const int Ho = resize ? 299 : H, Wo = resize ? 299 : W;
    return launch_k(k_inc_input, dim3(inc_grid((long long)N * Ho * Wo)), dim3(256), 0, st, x, N, H, W, Ho, Wo, resize, normalize, out);
}

// ------------------------------------------------------------------------------------------------ host side: the forward
// One walk over the network serves both the sizing (dry: records each buffer's largest use and checks every shape) and the
// launches.  Buffers (NHWC fp32): X the input, A / B the trunk (a block reads one and writes the other), T0 / T1 the branch
// intermediates, T2 the pooled input of a branch_pool conv.
struct IncWalk {
    enum { X, A, B, T0, T1, T2, NBUF };
    bool dry = true;
    int N = 0;
    long long need[NBUF] = {};                 // floats
    float* buf[NBUF] = {};
    const float* packed = nullptr;
    cudaStream_t st = nullptr;
    cudaError_t err = cudaSuccess;
    const char* bad = nullptr;                 // a shape the network cannot take (dry)
    int step = 0;                              // convs launched so far
    int (*layout)[4] = nullptr;                // dry, optional: per conv {c_off, C_total, writes the trunk (A / B), step}
    float* spatial = nullptr;                  // optional: sFID's [N][H W INC_SPATIAL_C] features of Mixed_6d (see spatial_tap)

    bool ok() const { return err == cudaSuccess && bad == nullptr; }
    void use(int b, int H, int W, int C) {
        const long long n = (long long)N * H * W * C;
        if ((long long)N * H * W > INT_MAX) bad = "N * H * W of an activation exceeds 2^31 - 1";
        if (n > need[b]) need[b] = n;
    }
    // conv i of the table reads buffer `src` [H][W][cin] and writes channels [c_off, +cout) of `dst` [Ho][Wo][C_total]
    void conv(int i, int src, int H, int W, int dst, int c_off, int C_total, int& Ho, int& Wo) {
        const IncConv& c = inc_convs()[i];
        Ho = inc_conv_out(H, c.kh, c.stride, c.ph); Wo = inc_conv_out(W, c.kw, c.stride, c.pw);
        if (dry) {
            if (Ho < 1 || Wo < 1) bad = "the input is too small for the requested block (a convolution has an empty output)";
            use(dst, Ho, Wo, C_total);
            if (layout) { layout[i][0] = c_off; layout[i][1] = C_total; layout[i][2] = dst == A || dst == B; layout[i][3] = step; }
        } else if (ok()) {
            const long long* o = &inc_packed_offsets()[2 * i];
            err = inc_conv_launch(c, buf[src], N, H, W, packed + o[0], packed + o[1], buf[dst], c_off, C_total, st);
        }
        ++step;
    }
    void conv(int i, int src, int H, int W, int dst, int c_off, int C_total) { int a, b; conv(i, src, H, W, dst, c_off, C_total, a, b); }
    void pool(int kind, int src, int H, int W, int C, int dst, int c_off, int C_total, int& Ho, int& Wo) {
        inc_pool_dims(kind, H, W, Ho, Wo);
        if (dry) {
            if (Ho < 1 || Wo < 1) bad = "the input is too small for the requested block (a max pool has an empty output)";
            use(dst, Ho, Wo, C_total);
        } else if (ok()) {
            err = inc_pool_launch(kind, buf[src], N, H, W, C, buf[dst], c_off, C_total, st);
        }
    }
    // buffer `src` [H][W][C] holds Mixed_6d's output: gather sFID's features into `spatial` (nothing when it is null)
    void spatial_tap(int src, int H, int W, int C) {
        if (dry || !spatial || !ok()) return;
        const long long pixels = (long long)N * H * W;
        err = launch_k(k_sfid_gather, dim3(inc_grid(pixels * INC_SPATIAL_C)), dim3(256), 0, st, buf[src], pixels, C, spatial);
    }
};

// Walks blocks 0..last_block in the order the torch forward runs the layers (the FID A, C and E blocks compute branch1x1 inside
// their torch.cat, after the other branches; conv indices are state_dict positions).  `emit(block, buffer, H, W, C)` is called
// at the end of each block with its NHWC output (block 3: before the global average).
template <typename Emit>
inline void inc_walk(IncWalk& w, int H, int W, int resize, int last_block, Emit&& emit) {
    enum { X = IncWalk::X, A = IncWalk::A, B = IncWalk::B, T0 = IncWalk::T0, T1 = IncWalk::T1, T2 = IncWalk::T2 };
    w.step = 0;
    const int Hi = resize ? 299 : H, Wi = resize ? 299 : W;
    if (w.dry) w.use(X, Hi, Wi, 12);
    int h = Hi, wd = Wi, h2, w2;
    w.conv(0, X, h, wd, A, 0, 32, h2, w2); h = h2; wd = w2;
    w.conv(1, A, h, wd, B, 0, 32, h2, w2); h = h2; wd = w2;
    w.conv(2, B, h, wd, A, 0, 64, h2, w2);
    w.pool(INC_MAX3_S2, A, h, wd, 64, B, 0, 64, h2, w2); h = h2; wd = w2;
    emit(0, B, h, wd, 64);
    if (last_block == 0 || !w.ok()) return;
    w.conv(3, B, h, wd, A, 0, 80);
    w.conv(4, A, h, wd, B, 0, 192, h2, w2); h = h2; wd = w2;
    w.pool(INC_MAX3_S2, B, h, wd, 192, A, 0, 192, h2, w2); h = h2; wd = w2;
    emit(1, A, h, wd, 192);
    if (last_block == 1 || !w.ok()) return;
    int cur = A, nxt = B, cin = 192, ho, wo, i = 5;
    for (int pf : {32, 64, 64}) {                                        // Mixed_5b..5d (A blocks)
        const int ct = 224 + pf;
        w.conv(i + 1, cur, h, wd, T0, 0, 48); w.conv(i + 2, T0, h, wd, nxt, 64, ct);
        w.conv(i + 3, cur, h, wd, T0, 0, 64); w.conv(i + 4, T0, h, wd, T1, 0, 96); w.conv(i + 5, T1, h, wd, nxt, 128, ct);
        w.conv(i, cur, h, wd, nxt, 0, ct);
        w.pool(INC_AVG3_S1, cur, h, wd, cin, T2, 0, cin, ho, wo); w.conv(i + 6, T2, h, wd, nxt, 224, ct);
        std::swap(cur, nxt); cin = ct; i += 7;
    }
    // Mixed_6a (B block)
    w.conv(i, cur, h, wd, nxt, 0, 768, ho, wo);
    w.conv(i + 1, cur, h, wd, T0, 0, 64); w.conv(i + 2, T0, h, wd, T1, 0, 96); w.conv(i + 3, T1, h, wd, nxt, 384, 768);
    w.pool(INC_MAX3_S2, cur, h, wd, 288, nxt, 480, 768, h2, w2);
    std::swap(cur, nxt); h = ho; wd = wo; i += 4;
    const int c7s[4] = {128, 160, 160, 192};
    for (int k = 0; k < 4; ++k) {                                        // Mixed_6b..6e (C blocks)
        const int c7 = c7s[k];
        w.conv(i + 1, cur, h, wd, T0, 0, c7); w.conv(i + 2, T0, h, wd, T1, 0, c7); w.conv(i + 3, T1, h, wd, nxt, 192, 768);
        w.conv(i + 4, cur, h, wd, T0, 0, c7); w.conv(i + 5, T0, h, wd, T1, 0, c7); w.conv(i + 6, T1, h, wd, T0, 0, c7);
        w.conv(i + 7, T0, h, wd, T1, 0, c7); w.conv(i + 8, T1, h, wd, nxt, 384, 768);
        w.conv(i, cur, h, wd, nxt, 0, 768);
        w.pool(INC_AVG3_S1, cur, h, wd, 768, T2, 0, 768, ho, wo); w.conv(i + 9, T2, h, wd, nxt, 576, 768);
        std::swap(cur, nxt); i += 10;
        if (k == 2) w.spatial_tap(cur, h, wd, 768);                     // Mixed_6d, before Mixed_7a overwrites this buffer
    }
    emit(2, cur, h, wd, 768);
    if (last_block == 2 || !w.ok()) return;
    // Mixed_7a (D block)
    w.conv(i, cur, h, wd, T0, 0, 192); w.conv(i + 1, T0, h, wd, nxt, 0, 1280, ho, wo);
    w.conv(i + 2, cur, h, wd, T0, 0, 192); w.conv(i + 3, T0, h, wd, T1, 0, 192); w.conv(i + 4, T1, h, wd, T0, 0, 192);
    w.conv(i + 5, T0, h, wd, nxt, 320, 1280);
    w.pool(INC_MAX3_S2, cur, h, wd, 768, nxt, 512, 1280, h2, w2);
    std::swap(cur, nxt); h = ho; wd = wo; cin = 1280; i += 6;
    for (int kind : {INC_AVG3_S1, INC_MAX3_S1}) {                         // Mixed_7b, 7c (E blocks)
        w.conv(i + 1, cur, h, wd, T0, 0, 384); w.conv(i + 2, T0, h, wd, nxt, 320, 2048); w.conv(i + 3, T0, h, wd, nxt, 704, 2048);
        w.conv(i + 4, cur, h, wd, T0, 0, 448); w.conv(i + 5, T0, h, wd, T1, 0, 384); w.conv(i + 6, T1, h, wd, nxt, 1088, 2048);
        w.conv(i + 7, T1, h, wd, nxt, 1472, 2048);
        w.conv(i, cur, h, wd, nxt, 0, 2048);
        w.pool(kind, cur, h, wd, cin, T2, 0, cin, ho, wo); w.conv(i + 8, T2, h, wd, nxt, 1856, 2048);
        std::swap(cur, nxt); cin = 2048; i += 9;
    }
    emit(3, cur, h, wd, 2048);
}

inline size_t inc_al256(size_t b) { return (b + 255) & ~size_t(255); }

// dry walk: per-buffer sizes; returns the workspace bytes, or 0 with `why` set when the shape is refused
inline size_t inc_workspace(int N, int H, int W, int resize, int last_block, IncWalk& w, const char*& why) {
    w = IncWalk();
    w.dry = true; w.N = N;
    inc_walk(w, H, W, resize, last_block, [](int, int, int, int, int) {});
    why = w.bad;
    if (w.bad) return 0;
    size_t total = 0;
    for (int b = 0; b < IncWalk::NBUF; ++b) total += inc_al256((size_t)w.need[b] * 4);
    return total;
}

}  // namespace ddpm
