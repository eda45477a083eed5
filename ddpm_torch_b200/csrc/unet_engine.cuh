// UNet plan builder + executor.  The network of ddpm_torch/models/unet.py:92-233 is compiled once per
// (batch, resolution) into flat lists of kernel launches (pack / forward / backward) over a caller-owned workspace.
// The backward list is produced tape-style: every forward block registers a closure that appends its adjoint ops.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>
#include "gemm_build.cuh"
#include "conv_halo.cuh"
#include "conv_halo.cuh"
#include "attn_fused.cuh"
#include "kernels_simt.cuh"

namespace ddpm {

struct ParamInfo { std::string name; int nd; int dims[4]; long long numel; long long off; };
struct T4 { long long off = -1; int B = 0, H = 0, W = 0, C = 0;
            long long qs = -1;    // workspace offset of the producer-written quad statistics [B][C/4][2] fp64 (-1: none)
            long long pix() const { return (long long)B * H * W; } long long numel() const { return pix() * C; } };
struct Src { T4 t0, t1; bool two = false; int C() const { return t0.C + (two ? t1.C : 0); } };
enum { OP_TEMB = 1 };
// Role of a backward op, which decides whether it runs in a given backward variant (ddpm_unet_backward_ex):
//   DATA   on the path from d_eps to the activation gradients: always runs
//   PARAM  only feeds the flat gradient buffer (weight gradients, bias column sums, gradient unpacks, the timestep MLP): skipped
//          when no parameter gradients are asked for
//   MIXED  produces activation gradients and also writes parameter gradients (GroupNorm dgamma/dbeta and fused column sums, the
//          gradient-buffer memset): always runs, and drops its flat-buffer writes when no parameter gradients are asked for
//   DX     the data gradient of in_conv (d_eps -> dx of the network input): runs only when dx is asked for
enum { ROLE_DATA = 0, ROLE_PARAM = 1, ROLE_MIXED = 2, ROLE_DX = 3 };
struct Op { std::string name; double flops; std::function<int(cudaStream_t)> run; int launches = 1; bool side = false; int tag = 0;
            int wait_pack = 0;   // forward list: 1 = needs the packed timestep-MLP weights, 2 = first consumer of the packed conv weights
            int chunk = -1;   // >= 0: gradient-chunk boundary of the backward list (see UnetEngine::chunks)
            int role = ROLE_DATA;
            bool runs(bool want_dx, bool param_grads) const { return role == ROLE_DX ? want_dx : (role == ROLE_PARAM ? param_grads : true); }
};
// A contiguous range [lo, hi) of the flat gradient buffer that is FINAL once `ev` has fired (recorded by the backward pass on the
// side stream, after the last weight-gradient GEMM / gradient unpack / main-chain reduction that writes into it).  Chunks are
// listed in the order the backward completes them, so a data-parallel caller can start the all-reduce of a chunk while the
// rest of the backward is still running (utils/train.py:149-153 does this with DDP's buckets).
struct GradChunk { long long lo = 0, hi = 0; int unpack_lo = 0, unpack_hi = 0; cudaEvent_t ev = nullptr; };
struct GnSaved { Src in; float* K; const float* gamma; const float* beta; float* dgamma; float* dbeta; int silu; float drop_p; uint32_t layer; unsigned char* mask; };

static inline int grid_for(long long n, int threads = 256) { long long g = (n + threads - 1) / threads; if (g > kPlanSms * 16) g = kPlanSms * 16; if (g < 1) g = 1; return (int)g; }
static inline int oct_threads(int C) { const int oct = C / 8; return oct <= 256 ? (256 / oct) * oct : 0; }

// ------------------------------------------------------------------ GroupNorm / column-sum launches
// Shared by the engine's plans and the GroupNorm operators of the C ABI, so that both launch the same geometry.
// The GroupNorm kernels give every thread one channel octet of the concat for its whole pixel loop: at most 256 octets.
constexpr int kGnMaxC = 2048;
// blocks over the pixels of one image: keep the whole launch within one wave of (kPlanSms x occ) CTAs
static inline void gn_grid(int Bn, int HW, int occ, int& nblk, int& ppb) {
    nblk = (kPlanSms * occ) / Bn; if (nblk > HW / 16) nblk = HW / 16; if (nblk < 1) nblk = 1;
    ppb = (HW + nblk - 1) / nblk; nblk = (HW + ppb - 1) / ppb;
}
// Grid granularity (DDPM_GN_STATS_OCC / _APPLY_OCC / _BWD_OCC override it): blocks per image = kPlanSms*occ/B with occ 4 -
// finer grids pay more per-block prologue / atomics than the wave-quantisation they would save.
static inline int gn_occ(const char* env) { const char* v = getenv(env); return v ? atoi(v) : 4; }
// k_gn_stats: fp64 {sum, sumsq} per (image, group) into the zeroed stats[B][64]; the last block of an image writes fin.K
static inline int launch_gn_stats(const GnSrc& s, double* stats, int Bn, int HW, const GnFin& fin, cudaStream_t st) {
    static const int occ = gn_occ("DDPM_GN_STATS_OCC");
    int nblk, ppb; gn_grid(Bn, HW, occ, nblk, ppb);
    launch_k(k_gn_stats, dim3(nblk, Bn), oct_threads(s.C0 + s.C1), 0, st, s, stats, HW, ppb, fin);
    return (int)cudaGetLastError();
}
// k_gn_apply: y = act(x*sc + sh) [* dropout], sc/sh from a.K, or from the producers' quad statistics when a.qs0 is set
static inline int launch_gn_apply(const GnApply& a, int Bn, cudaStream_t st) {
    static const int occ = gn_occ("DDPM_GN_APPLY_OCC");
    int nblk, ppb; gn_grid(Bn, a.HW, occ, nblk, ppb);
    launch_k(k_gn_apply, dim3(nblk, Bn), oct_threads(a.s.C0 + a.s.C1), 0, st, a, ppb);
    return (int)cudaGetLastError();
}
// k_gn_small: statistics + apply in one launch, one block per image (HW <= 64)
static inline int launch_gn_small(const GnApply& a, int Bn, cudaStream_t st) {
    launch_k(k_gn_small, Bn, oct_threads(a.s.C0 + a.s.C1), 0, st, a);
    return (int)cudaGetLastError();
}
// k_gn_prep: a.Kout from the producers' quad statistics, no pass over the tensor
static inline int launch_gn_prep(const GnApply& a, int Bn, cudaStream_t st) {
    const int C = a.s.C0 + a.s.C1;
    launch_k(k_gn_prep, Bn, C < 256 ? C : 256, 0, st, a);
    return (int)cudaGetLastError();
}
// ------------------------------------------------------------------ bits/dim launches
// Shared by ddpm_bpd_step (through the plan's out_conv.2.gather op or the tail after the forward) and the bits/dim operator of
// the C ABI (ddpm_bpd_terms_run), so that both launch the same kernels on the same grid: one 256-thread block per 256 pixels
// of one image, blocks never straddling images (kernels_simt.cuh).
static inline int bpd_blocks(int Bn, int HW) { return Bn * ((HW + 255) / 256); }
// k_out_gather<Cout>, Cout 1..3: the bits/dim grid when bp.part is set, else the caller's grid-stride grid nblk
static inline int launch_out_gather(int Cout, int nblk, cudaStream_t st, const float* T, const float* bias, float* out, int Bn, int Hn,
                                    int Wn, const PsampleEpi& ps, const BpdEpi& bp) {
    const int g = bp.part ? bpd_blocks(Bn, Hn * Wn) : nblk;
    switch (Cout) {
        case 1: launch_k(k_out_gather<1>, g, 256, 0, st, T, bias, out, Bn, Hn, Wn, ps, bp); break;
        case 2: launch_k(k_out_gather<2>, g, 256, 0, st, T, bias, out, Bn, Hn, Wn, ps, bp); break;
        default: launch_k(k_out_gather<3>, g, 256, 0, st, T, bias, out, Bn, Hn, Wn, ps, bp); break;
    }
    return (int)cudaGetLastError();
}
// k_bpd_tail<Cout>, Cout 1..4, over eps f32 [Bn][Cout][HW]
static inline int launch_bpd_tail(int Cout, cudaStream_t st, const float* eps, const BpdEpi& bp, int Bn, int HW) {
    const int g = bpd_blocks(Bn, HW);
    switch (Cout) {
        case 1: launch_k(k_bpd_tail<1>, g, 256, 0, st, eps, bp, HW); break;
        case 2: launch_k(k_bpd_tail<2>, g, 256, 0, st, eps, bp, HW); break;
        case 3: launch_k(k_bpd_tail<3>, g, 256, 0, st, eps, bp, HW); break;
        default: launch_k(k_bpd_tail<4>, g, 256, 0, st, eps, bp, HW); break;
    }
    return (int)cudaGetLastError();
}
// k_bpd_finalize over the bpd_blocks(Bn, HW) partials: losses / mses [Bn][T], column coef[kBpdRow]
static inline int launch_bpd_finalize(cudaStream_t st, const float* part, int Bn, int Cout, int HW, const float* coef, int T,
                                      float* losses, float* mses) {
    launch_k(k_bpd_finalize, 1, 256, 0, st, part, (HW + 255) / 256, Bn, (float)(Cout * HW), coef, T, losses, mses);
    return (int)cudaGetLastError();
}
// dropout is armed per call by a non-zero seed
static inline void gn_arm_dropout(float& drop_p, unsigned long long& seed, unsigned long long run_seed) { seed = run_seed; if (!seed) drop_p = 0.f; }
// k_gn_bwd_reduce + k_gn_bwd_apply; the apply pass also accumulates the column sums of dx when any of the cs pointers is set
static inline int launch_gn_bwd(const GnBwd& a0, float* cs_per_img, int cs_ld, float* cs_total, float* cs_total2, cudaStream_t st) {
    static const int occ = gn_occ("DDPM_GN_BWD_OCC");
    GnBwd a = a0;
    int nblk; gn_grid(a.B, a.HW, occ, nblk, a.pix_per_block);
    const int C = a.s.C0 + a.s.C1, thr = oct_threads(C);
    const dim3 g(nblk, a.B);
    launch_k(k_gn_bwd_reduce, g, thr, (size_t)2 * C * 4, st, a);
    if (cs_per_img || cs_total || cs_total2) launch_k(k_gn_bwd_apply<true>, g, thr, (size_t)C * 4, st, a, cs_per_img, cs_ld, cs_total, cs_total2);
    else                                     launch_k(k_gn_bwd_apply<false>, g, thr, 0, st, a, cs_per_img, cs_ld, cs_total, cs_total2);
    return (int)cudaGetLastError();
}
// k_colsum over dy [B][HW][C]: column sums of the first C_valid channels; C above kGnMaxC runs as kGnMaxC-wide slices in grid z
static inline int launch_colsum(const bf16* dy, float* per_img, int ld, float* total, float* total2, int Bn, int HW, int C, int C_valid,
                                cudaStream_t st) {
    const int cs = C < kGnMaxC ? C : kGnMaxC, nz = (C + cs - 1) / cs;
    int nblk = (592 + Bn - 1) / Bn; if (nblk > HW / 8) nblk = HW / 8; if (nblk < 1) nblk = 1;
    const int ppb = (HW + nblk - 1) / nblk; nblk = (HW + ppb - 1) / ppb;
    launch_k(k_colsum, dim3(nblk, Bn, nz), oct_threads(cs), (size_t)cs * 4, st, dy, per_img, ld, total, total2, HW, C, C_valid, ppb, cs);
    return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ attention core launches
// softmax(Q K^T / sqrt(C)) V of AttentionBlock (unet.py:43-51) and its backward, with qkv bf16 [NB][T][3C].  Shared by the engine's
// plans (attn_block) and the attention operators of the C ABI: a route is built as a list of launch steps, which the engine pushes
// as ops named <block> + step.name and the operators run in order, so both launch the same kernels with the same grids.
//   1 fused     T = 256, C = 256: attn_kernel<false> (attn_fused.cuh); backward attn_kernel<true> + the dV / dK products
//   2 t16       T = 16, C in {128, 256, 512}: k_attn16_fwd / k_attn16_bwd, one CTA per image
//   3 products  Q.K^T -> k_softmax_rows -> P.V; backward dP, dV, k_softmax_bwd, dQ, dK.  The products run on the GEMM engine when
//               attn_bmm_tc(T, C), on CUDA cores (k_sgemm) otherwise
enum { ATTN_ROUTE_FUSED = 1, ATTN_ROUTE_T16 = 2, ATTN_ROUTE_PRODUCTS = 3 };
enum { ATTN_STEP_AUX = 0, ATTN_STEP_TC = 1, ATTN_STEP_SIMT = 2 };   // what a step counts as in the plan statistics
struct AttnStep { std::string name; double flops; int kind; std::function<int(cudaStream_t)> run; };
using AttnSteps = std::vector<AttnStep>;

// the products of route 3 take the GEMM engine for a power-of-two T that is a multiple of 128 and C % 64 == 0
inline bool attn_bmm_tc(int T, int Cc) { return (T % 128 == 0) && (Cc % 64 == 0) && ((T & (T - 1)) == 0); }

// k_attn16_* need attn16_smem(512, .) bytes of dynamic shared memory at C = 512: raise the limit once per device.  The engine calls
// this at plan time, so that no launch of a plan (which may be under graph capture) has to
inline int attn16_prepare() {
    static unsigned done = 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 32 && ((done >> dev) & 1u)) return 0;
    e = cudaFuncSetAttribute(k_attn16_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn16_smem(512, false));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_attn16_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn16_smem(512, true));
    if (e != cudaSuccess) return (int)e;
    if (dev < 32) done |= 1u << dev;
    return 0;
}
static inline int launch_attn16_fwd(const bf16* qkv, bf16* O, bf16* P, int NB, int C, float scale, cudaStream_t st) {
    const int rc = attn16_prepare(); if (rc) return rc;
    launch_k(k_attn16_fwd, NB, 256, attn16_smem(C, false), st, qkv, O, P, C, scale);
    return (int)cudaGetLastError();
}
static inline int launch_attn16_bwd(const bf16* qkv, const bf16* dO, const bf16* P, bf16* dqkv, int NB, int C, float scale, cudaStream_t st) {
    const int rc = attn16_prepare(); if (rc) return rc;
    launch_k(k_attn16_bwd, NB, 256, attn16_smem(C, true), st, qkv, dO, P, dqkv, C, scale);
    return (int)cudaGetLastError();
}
// one warp per row of [rows][T]
static inline int launch_softmax_rows(const float* S, bf16* P, long long rows, int T, cudaStream_t st) {
    launch_k(k_softmax_rows, (int)((rows + 7) / 8), 256, 0, st, S, P, rows, T);
    return (int)cudaGetLastError();
}
static inline int launch_softmax_bwd(const bf16* P, const float* dP, bf16* dS, long long rows, int T, float scale, cudaStream_t st) {
    launch_k(k_softmax_bwd, (int)((rows + 7) / 8), 256, 0, st, P, dP, dS, rows, T, scale);
    return (int)cudaGetLastError();
}

// Batched matmuls of the attention block (unet.py:43-51) and their adjoints.
//   form 0 (NT): C[b][i][j] = alpha * sum_c A[b][i][c] * B[b][j][c]     M=i, N=j, K=c
//   form 1 (NN): C[b][i][c] = sum_j A[b][i][j] * B[b][j][c]             M=i, N=c, K=j
//   form 2 (TN): C[b][j][c] = sum_i A[b][i][j] * B[b][i][c]             M=j, N=c, K=i
// A, B bf16 with row strides lda/ldb and per-batch strides = rows*ld; C bf16 or fp32.  A dry plan builds no tensor maps: its
// tensor-core step does nothing.
inline int attn_bmm(AttnSteps& S, const std::string& name, int form, const bf16* A, long long lda, long long sa,
                    const bf16* Bp, long long ldb, long long sb, void* C, long long ldc, long long sc, bool c_f32,
                    int nb, int T, int Cc, float alpha, bool dry) {
    // all attention products here are T x T x Cc shaped
    const int M = T, N = (form == 0) ? T : Cc, K = (form == 0) ? Cc : T;
    const double fl = 2.0 * nb * (double)M * N * K;
    if (attn_bmm_tc(T, Cc)) {
        ddpm_gemm_desc d; memset(&d, 0, sizeof d);
        d.M = M; d.N = N; d.W = T; d.H = 1; d.NB = nb; d.alpha = alpha; d.grid_z = nb;
        d.out = C; d.ldo = (int)ldc; d.out_z_stride = sc; d.flags = c_f32 ? EPI_OUT_F32 : 0;
        d.a_ptr[0] = A; d.a_ld[0] = lda;
        if (form == 0) {
            d.mode = GEMM_KK; d.a_C[0] = K; d.nseg = 1; d.seg_map[0] = 0; d.seg_taps[0] = 1; d.seg_kchunks[0] = K / 64; d.seg_cbase[0] = 0;
            d.b_ptr = Bp; d.b_K = K; d.b_rows = N; d.b_batch = nb; d.b_ld = ldb; d.b_bs = sb; d.a_z_n = 1; d.b_z = 1;
        } else if (form == 1) {
            d.mode = GEMM_KMN; d.a_C[0] = K; d.b_ptr = Bp; d.b_K = N; d.b_ld = ldb; d.kblocks = K / 64; d.a_z_n = 1;
        } else {
            d.mode = GEMM_MNMN; d.a_C[0] = M; d.b_ptr = Bp; d.b_K = N; d.b_ld = ldb; d.taps = 1; d.splits = 1; d.kblocks = K / 64;
        }
        if (dry) { S.push_back({name, fl, ATTN_STEP_TC, [](cudaStream_t) { return 0; }}); return 0; }
        GemmLaunch g; const int rc = build_gemm(d, g);
        if (rc) return rc;
        S.push_back({name, fl, ATTN_STEP_TC, [g](cudaStream_t st) { return launch_gemm(g, st); }});
        return 0;
    }
    SgemmParams p; memset(&p, 0, sizeof p);
    p.A = A; p.B = Bp; p.C = C; p.M = M; p.N = N; p.K = K; p.alpha = alpha;
    p.sa_z = sa; p.sb_z = sb; p.sc_z = sc; p.sc_m = ldc; p.sc_n = 1;
    if (form == 0) { p.sa_m = lda; p.sa_k = 1; p.sb_k = 1; p.sb_n = ldb; }
    else if (form == 1) { p.sa_m = lda; p.sa_k = 1; p.sb_k = ldb; p.sb_n = 1; }
    else { p.sa_m = 1; p.sa_k = lda; p.sb_k = ldb; p.sb_n = 1; }
    const dim3 grid((N + 63) / 64, (M + 63) / 64, nb);
    if (c_f32) S.push_back({name + "[simt]", fl, ATTN_STEP_SIMT, [p, grid](cudaStream_t st) { launch_k(k_sgemm<bf16, bf16, float>, grid, 256, 0, st, p); return (int)cudaGetLastError(); }});
    else       S.push_back({name + "[simt]", fl, ATTN_STEP_SIMT, [p, grid](cudaStream_t st) { launch_k(k_sgemm<bf16, bf16, bf16>, grid, 256, 0, st, p); return (int)cudaGetLastError(); }});
    return 0;
}

// forward of `route`: O bf16 [NB][T][C]; P bf16 [NB][T][T] (routes 1 and 2: written when not null; route 3: always);
// S fp32 [NB][T][T] (route 3 only)
inline int attn_fwd_steps(AttnSteps& out, int route, const bf16* qkv, bf16* O, bf16* P, float* S, int NB, int T, int C, bool dry) {
    const float scale = 1.f / sqrtf((float)C);
    const long long ldq = 3 * C, sq = (long long)T * 3 * C, tt = (long long)T * T;
    const double fl = 4.0 * NB * (double)T * T * C;
    if (route == ATTN_ROUTE_FUSED) {
        // Q.K^T -> softmax -> P.V in ONE kernel, S and O in registers, P in shared memory (attn_fused.cuh)
        if (dry) { out.push_back({".attn[fused]", fl, ATTN_STEP_TC, [](cudaStream_t) { return 0; }}); return 0; }
        AttnLaunch g; const int rc = build_attn(qkv, O, NB, T, C, g, P);
        if (rc) return rc;
        out.push_back({".attn[fused]", fl, ATTN_STEP_TC, [g](cudaStream_t st) { return launch_attn(g, st); }});
        return 0;
    }
    if (route == ATTN_ROUTE_T16) {
        // 4x4 level: one CTA per image does scores, softmax and P.V
        out.push_back({".attn[t16]", fl, ATTN_STEP_SIMT, [=](cudaStream_t st) { return launch_attn16_fwd(qkv, O, P, NB, C, scale, st); }});
        return 0;
    }
    int rc = attn_bmm(out, ".qk", 0, qkv, ldq, sq, qkv + C, ldq, sq, S, T, tt, true, NB, T, C, scale, dry);
    if (rc) return rc;
    const long long rows = (long long)NB * T;
    out.push_back({".softmax", 0, ATTN_STEP_AUX, [=](cudaStream_t st) { return launch_softmax_rows(S, P, rows, T, st); }});
    return attn_bmm(out, ".pv", 1, P, T, tt, qkv + 2 * C, ldq, sq, O, C, (long long)T * C, false, NB, T, C, 1.f, dry);
}

// backward of `route` from the P its forward wrote: dO bf16 [NB][T][C] -> all three thirds of dqkv bf16 [NB][T][3C].
// dS bf16 [NB][T][T] (routes 1 and 3) and dP fp32 [NB][T][T] (route 3) are intermediates the route materialises
inline int attn_bwd_steps(AttnSteps& out, int route, const bf16* qkv, const bf16* dO, const bf16* P, float* dP, bf16* dS, bf16* dqkv,
                          int NB, int T, int C, bool dry) {
    const float scale = 1.f / sqrtf((float)C);
    const long long ldq = 3 * C, sq = (long long)T * 3 * C, tt = (long long)T * T, so = (long long)T * C;
    if (route == ATTN_ROUTE_T16) {
        const double fl = 8.0 * NB * (double)T * T * C;
        out.push_back({".attn_bwd[t16]", fl, ATTN_STEP_SIMT, [=](cudaStream_t st) { return launch_attn16_bwd(qkv, dO, P, dqkv, NB, C, scale, st); }});
        return 0;
    }
    int rc;
    if (route == ATTN_ROUTE_FUSED) {
        // dP -> softmax backward -> dQ in one launch (attn_kernel<true>); dK and dV read dS / P back as GEMM operands
        const double fl = 4.0 * NB * (double)T * T * C;
        if (dry) out.push_back({".attn_bwd[fused]", fl, ATTN_STEP_TC, [](cudaStream_t) { return 0; }});
        else {
            AttnLaunch g;
            if ((rc = build_attn_bwd(qkv, dO, P, dS, dqkv, NB, T, C, g))) return rc;
            out.push_back({".attn_bwd[fused]", fl, ATTN_STEP_TC, [g](cudaStream_t st) { return launch_attn_bwd(g, st); }});
        }
        if ((rc = attn_bmm(out, ".dV", 2, P, T, tt, dO, C, so, dqkv + 2 * C, ldq, sq, false, NB, T, C, 1.f, dry))) return rc;
        return attn_bmm(out, ".dK", 2, dS, T, tt, qkv, ldq, sq, dqkv + C, ldq, sq, false, NB, T, C, 1.f, dry);
    }
    if ((rc = attn_bmm(out, ".dP", 0, dO, C, so, qkv + 2 * C, ldq, sq, dP, T, tt, true, NB, T, C, 1.f, dry))) return rc;
    if ((rc = attn_bmm(out, ".dV", 2, P, T, tt, dO, C, so, dqkv + 2 * C, ldq, sq, false, NB, T, C, 1.f, dry))) return rc;
    const long long rows = (long long)NB * T;
    out.push_back({".softmax_bwd", 0, ATTN_STEP_AUX, [=](cudaStream_t st) { return launch_softmax_bwd(P, dP, dS, rows, T, scale, st); }});
    if ((rc = attn_bmm(out, ".dQ", 1, dS, T, tt, qkv + C, ldq, sq, dqkv, ldq, sq, false, NB, T, C, 1.f, dry))) return rc;
    return attn_bmm(out, ".dK", 2, dS, T, tt, qkv, ldq, sq, dqkv + C, ldq, sq, false, NB, T, C, 1.f, dry);
}

// ------------------------------------------------------------------ convolution launches
// The convolutions of the plans (conv_op, wgrad_op, the stride-2 data gradient of down_conv, the folded upsample of up_conv) and
// the conv operator of the C ABI (ddpm_conv_run) are built by the functions below, so that both launch the same kernels with the
// same descriptors, block_n and split counts over weights packed by the same PackEntry rows.  Routes:
//   1 halo  3x3 stride 1 (+ fused 1x1 skip segments): conv_halo.cuh.  conv_route_tc + halo_eligible
//   2 gemm  implicit GEMM on the tensor cores (GEMM_KK); split over K into a zeroed fp32 scratch + k_splitk_finalize when few output
//           tiles; weight gradients GEMM_MNMN with fp32 atomics
//   3 simt  k_conv_generic (+ a second launch for a skip), k_wgrad_generic: concat inputs, odd widths, MAP_TRANSPOSED2
//   4 s2    stride-2 3x3 on the tensor cores: forward (a_estride 2), data gradient as four output-parity GEMMs (PK_CONV dkind 3),
//           weight gradient (b_estride 2)
//   5 fold  nearest-2x upsample folded into the 3x3 conv that follows it: four output-parity GEMMs over PK_UPFOLD weights
enum { CONV_ROUTE_HALO = 1, CONV_ROUTE_GEMM = 2, CONV_ROUTE_SIMT = 3, CONV_ROUTE_S2 = 4, CONV_ROUTE_FOLD = 5 };
// a launch step; kind counts as in AttnStep (tensor-core op, CUDA-core op, or neither: the skip launch of the CUDA-core route)
struct ConvStep { std::string name; double flops; int kind; int launches; std::function<int(cudaStream_t)> run; };
using ConvSteps = std::vector<ConvStep>;

// Rows of the k_pack_table tables that lay out conv weights from the fp32 OIHW masters (the plans' repack and gradient unpack,
// and the conv operator).
//   PK_CONV      fwd [Co][ld_f] at column k_off (taps x Ci, tap-major) and / or dgr [Ci][ld_d] (dkind 1 plain, 2 flipped taps,
//                3 stride-2 parity blocks); either may be null
//   PK_IDENTITY  fwd[co][k_off + ci] = (co == ci)
//   PK_BIAS_ADD  dst = a + b
//   PK_UPFOLD    fwd [C][16C]: the nearest-2x upsample merged into the 3x3 weights, per output parity
//   PK_UNPACK_GRAD  scratch [9][Co][Ci] -> dw OIHW, scratch cleared behind the read
inline PackEntry pack_entry(int kind, int Co, int Ci, int taps) { PackEntry e; memset(&e, 0, sizeof e); e.kind = kind; e.Co = Co; e.Ci = Ci; e.taps = taps; return e; }
inline PackEntry pack_conv_entry(const float* w, int Co, int Ci, int taps, int k_off, bf16* fwd, long long ld_f, bf16* dgr, long long ld_d, int dkind) {
    PackEntry e = pack_entry(PK_CONV, Co, Ci, taps);
    e.k_off = k_off; e.w = w; e.fwd = fwd; e.ld_f = ld_f; e.dgr = dgr; e.ld_d = ld_d; e.dkind = dgr ? dkind : 0;
    return e;
}
inline PackEntry pack_identity_entry(bf16* fwd, long long ld_f, int k_off, int C) { PackEntry e = pack_entry(PK_IDENTITY, C, C, 1); e.k_off = k_off; e.fwd = fwd; e.ld_f = ld_f; return e; }
inline PackEntry pack_bias_add_entry(float* dst, const float* a, const float* b, int n) { PackEntry e = pack_entry(PK_BIAS_ADD, n, 1, 1); e.w = a; e.w2 = b; e.fout = dst; return e; }
inline PackEntry pack_upfold_entry(const float* w, int C, bf16* fwd, long long ld_f) { PackEntry e = pack_entry(PK_UPFOLD, C, C, 9); e.w = w; e.fwd = fwd; e.ld_f = ld_f; return e; }
inline PackEntry unpack_grad_entry(float* scratch, float* dw, int Co, int Ci) { PackEntry e = pack_entry(PK_UNPACK_GRAD, Co, Ci, 9); e.fout = dw; e.scratch = scratch; return e; }

// both box shapes the GEMM engine tiles NHWC maps with exist for an h x w map
inline bool conv_tc_geom(int h, int w) { int a, b, c; return pick_box(w, h, 128, a, b, c) && pick_box(w, h, 64, a, b, c); }

// out = conv(in) [+ 1x1 skip(skip)] + bias + rowvec[image] + residual, NHWC bf16 (accumulate: out += instead of a residual)
struct ConvArgs {
    GnSrc in{}; int B = 0, Hi = 0, Wi = 0;         // input concat (C1 = 0: one source) on an Hi x Wi map
    int ksize = 3, stride = 1, map = MAP_NORMAL;
    const bf16* wp = nullptr; long long ldw = 0;   // packed [Co][ldw]: taps x Cin, then the skip's K chunks
    bool has_skip = false, skip_identity = false;  // skip_identity: the skip chunks carry identity weights (no FLOPs counted)
    GnSrc skip{};
    const float* bias = nullptr; const float* rowvec = nullptr; int rowvec_ld = 0; const bf16* residual = nullptr;
    bf16* out = nullptr; int Co = 0, Ho = 0, Wo = 0; bool accumulate = false;
    double* qstats = nullptr;                      // quad statistics of the output (halo and single-pass GEMM routes)
    const float* xfK = nullptr; int xf_silu = 0;   // GroupNorm(+SiLU) folded into the operand path (halo route only)
    int Cin() const { return in.C0 + in.C1; }
    int skipC() const { return has_skip ? skip.C0 + skip.C1 : 0; }
};
struct ConvChoice { int route = 0; int block_n = 0; int splits = 1; bool n128 = false; };

// SamePad2d(3,2) + 3x3 stride 2 (unet.py:163-167) on the tensor cores: tap offsets 0..2 on the stride-2 sampled input
inline bool conv_s2_fwd(const ConvArgs& c) {
    return c.stride == 2 && c.map == MAP_NORMAL && c.ksize == 3 && !c.has_skip && c.Ho * 2 == c.Hi && c.Wo * 2 == c.Wi;
}
// the tensor-core routes (halo, gemm, s2) take one NHWC source with 64-channel chunks on a map the GEMM engine can tile
inline bool conv_route_tc(const ConvArgs& c) {
    const bool s2 = conv_s2_fwd(c);
    bool tc = (c.stride == 1 || s2) && c.map == MAP_NORMAL && c.in.C1 == 0 && c.in.C0 % 64 == 0 && c.Co % 64 == 0 &&
              (s2 || (c.Ho == c.Hi && c.Wo == c.Wi)) && conv_tc_geom(c.Ho, c.Wo) && !(c.accumulate && c.residual);
    if (c.has_skip) tc = tc && c.skip.C0 % 64 == 0 && c.skip.C1 % 64 == 0;
    return tc;
}
// The planner's choice for a conv.  allow_halo = false is DDPM_NO_HALO; n128_fill = false is DDPM_NO_N128_FILL.
inline ConvChoice conv_choose(const ConvArgs& c, bool allow_halo, bool n128_fill) {
    ConvChoice r;
    if (!conv_route_tc(c)) { r.route = CONV_ROUTE_SIMT; r.block_n = 64; return r; }
    if (allow_halo && c.ksize == 3 && c.stride == 1 && halo_eligible(c.Ho, c.Wo, c.Co)) { r.route = CONV_ROUTE_HALO; r.block_n = pick_block_n(c.Co); return r; }
    r.route = conv_s2_fwd(c) ? CONV_ROUTE_S2 : CONV_ROUTE_GEMM;
    // small-M problems (8x8 / 4x4 levels) do not fill the SMs with output tiles: split the K loop across CTAs
    // (fp32 atomics into a zeroed scratch) and finish bias / timestep vector / residual / bf16 in a tiny second kernel
    const long long Pout = (long long)c.B * c.Ho * c.Wo;
    int bn = pick_block_n(c.Co);
    int tiles = (int)((Pout + 127) / 128) * ((c.Co + bn - 1) / bn);
    // 8x8 levels: 64 tiles of 128x256 would need split-K (+ a finalize launch and fp32 atomics); 128 tiles of 128x128
    // fill the machine in one wave with the same MMA time per CTA and no second pass
    if (n128_fill && bn == 256 && tiles <= kPlanSms / 2 && tiles * 2 <= kPlanSms) { bn = 128; tiles *= 2; r.n128 = true; }
    const int slabs = (int)(((long long)c.ksize * c.ksize * c.Cin() + c.skipC()) / 64);
    int splits = 1;
    // (a finalize launch + fp32 atomics cost more than a half-empty single wave: split only when under ~1/3 of the SMs have a tile)
    if (tiles <= 48 && slabs >= 16) { splits = kPlanSms / tiles; if (splits > slabs / 8) splits = slabs / 8; if (splits > 16) splits = 16; if (splits < 1) splits = 1; }
    r.block_n = bn; r.splits = splits;
    return r;
}
inline double conv_flops(const ConvArgs& c) {
    const long long Pout = (long long)c.B * c.Ho * c.Wo;
    return 2.0 * Pout * c.Co * (double)(c.ksize * c.ksize * c.Cin() + (c.skip_identity ? 0 : c.skipC()));
}
// the launch steps of route ch.route; splitk_scratch: zeroed fp32 [B*Ho*Wo][Co] when ch.splits > 1 (left zeroed)
inline int conv_fwd_steps(ConvSteps& S, const ConvArgs& c, const ConvChoice& ch, float* splitk_scratch, bool dry) {
    const int Cin = c.Cin(), taps = c.ksize * c.ksize;
    const long long Pout = (long long)c.B * c.Ho * c.Wo;
    const double fl = conv_flops(c);
    const long long K = (long long)taps * Cin + c.skipC();
    const bf16* resid = c.accumulate ? c.out : c.residual;
    if (ch.route == CONV_ROUTE_HALO) {
        ddpm_halo_desc h; memset(&h, 0, sizeof h);
        h.NB = c.B; h.H = c.Ho; h.W = c.Wo; h.Cout = c.Co;
        h.a_ptr[0] = c.in.x0; h.a_C[0] = c.in.C0; h.a_ld[0] = c.in.C0;
        h.nseg = 1; h.seg_map[0] = 0; h.seg_taps[0] = 9; h.seg_kchunks[0] = c.in.C0 / 64; h.seg_cbase[0] = 0;
        if (c.has_skip) {
            h.a_ptr[1] = c.skip.x0; h.a_C[1] = c.skip.C0; h.a_ld[1] = c.skip.C0;
            h.seg_map[1] = 1; h.seg_taps[1] = 1; h.seg_kchunks[1] = c.skip.C0 / 64; h.seg_cbase[1] = 0; h.nseg = 2;
            if (c.skip.C1) {
                h.a_ptr[2] = c.skip.x1; h.a_C[2] = c.skip.C1; h.a_ld[2] = c.skip.C1;
                h.seg_map[2] = 2; h.seg_taps[2] = 1; h.seg_kchunks[2] = c.skip.C1 / 64; h.seg_cbase[2] = 0; h.nseg = 3;
            }
        }
        h.w = c.wp; h.ldw = c.ldw; h.Ktot = (int)K; h.out = c.out; h.bias = c.bias; h.rowvec = c.rowvec; h.rowvec_ld = c.rowvec_ld;
        h.residual = resid; h.base_offset_mode = 0; h.gn.qstats = c.qstats;
        if (c.xfK) { h.xf_K = c.xfK; h.xf_silu = c.xf_silu; h.force_sub = 3; }
        if (dry) { S.push_back({"[halo]", fl, ATTN_STEP_TC, 1, [](cudaStream_t) { return 0; }}); return 0; }
        HaloLaunch g; const int rc = build_halo(h, g);
        if (rc) return rc;
        S.push_back({"[halo]", fl, ATTN_STEP_TC, 1, [g](cudaStream_t st) { return launch_halo(g, st); }});
        return 0;
    }
    if (ch.route == CONV_ROUTE_GEMM || ch.route == CONV_ROUTE_S2) {
        ddpm_gemm_desc d; memset(&d, 0, sizeof d);
        d.mode = GEMM_KK; d.M = (int)Pout; d.N = c.Co; d.W = c.Wo; d.H = c.Ho; d.NB = c.B;
        d.a_ptr[0] = c.in.x0; d.a_C[0] = c.in.C0; d.a_ld[0] = c.in.C0;
        d.nseg = 1; d.seg_map[0] = 0; d.seg_taps[0] = taps; d.seg_kchunks[0] = c.in.C0 / 64; d.seg_cbase[0] = 0;
        if (ch.route == CONV_ROUTE_S2) {   // SamePad2d(3,2): pad bottom/right only -> tap offsets 0..2 on the stride-2 sampled map, OOB = zero fill
            d.a_estride = 2; d.seg_custom[0] = 1; d.seg_cmul[0] = 2;
            for (int t = 0; t < 9; ++t) { d.seg_dx[0][t] = (signed char)(t % 3); d.seg_dy[0][t] = (signed char)(t / 3); }
        }
        if (c.has_skip) {
            d.a_ptr[1] = c.skip.x0; d.a_C[1] = c.skip.C0; d.a_ld[1] = c.skip.C0;
            d.seg_map[1] = 1; d.seg_taps[1] = 1; d.seg_kchunks[1] = c.skip.C0 / 64; d.seg_cbase[1] = 0; d.nseg = 2;
            if (c.skip.C1) {
                d.a_ptr[2] = c.skip.x1; d.a_C[2] = c.skip.C1; d.a_ld[2] = c.skip.C1;
                d.seg_map[2] = 2; d.seg_taps[2] = 1; d.seg_kchunks[2] = c.skip.C1 / 64; d.seg_cbase[2] = 0; d.nseg = 3;
            }
        }
        d.b_ptr = c.wp; d.b_K = (int)K; d.b_rows = c.Co; d.b_batch = 1; d.b_ld = c.ldw; d.b_bs = 0;
        d.out = c.out; d.ldo = c.Co; d.alpha = 1.f; d.grid_z = 1;
        d.bias = c.bias; d.rowvec = c.rowvec; d.rowvec_ld = c.rowvec_ld; d.rows_per_vec = c.Ho * c.Wo;
        d.residual = resid; d.ldr = c.Co;
        if (ch.n128) d.block_n = 128;
        if (ch.splits > 1) {
            if (!splitk_scratch && !dry) return fail(-31, "internal: split-K conv without its scratch");
            ddpm_gemm_desc ds = d;
            ds.kk_splits = ch.splits; ds.grid_z = ch.splits; ds.out = splitk_scratch; ds.flags = EPI_OUT_F32 | EPI_ATOMIC;
            ds.bias = nullptr; ds.rowvec = nullptr; ds.residual = nullptr;
            if (dry) { S.push_back({"[splitk]", fl, ATTN_STEP_TC, 2, [](cudaStream_t) { return 0; }}); return 0; }
            const float* bias = c.bias; const float* rowvec = c.rowvec; const int rvld = c.rowvec_ld, rpv = c.Ho * c.Wo;
            float* scratch = splitk_scratch; bf16* outp = c.out;
            const long long M = Pout; const int N = c.Co; const int nfin = grid_for(M * (N / 8));
            GemmLaunch g; const int rc = build_gemm(ds, g);
            if (rc) return rc;
            S.push_back({"[splitk]", fl, ATTN_STEP_TC, 2, [=](cudaStream_t st) {
                const int r2 = launch_gemm(g, st); if (r2) return r2;
                launch_k(k_splitk_finalize, nfin, 256, 0, st, scratch, bias, rowvec, rvld, rpv, resid, outp, M, N);
                return (int)cudaGetLastError(); }});
            return 0;
        }
        d.gn.qstats = c.qstats;
        if (dry) { S.push_back({"", fl, ATTN_STEP_TC, 1, [](cudaStream_t) { return 0; }}); return 0; }
        GemmLaunch g; const int rc = build_gemm(d, g);
        if (rc) return rc;
        S.push_back({"", fl, ATTN_STEP_TC, 1, [g](cudaStream_t st) { return launch_gemm(g, st); }});
        return 0;
    }
    ConvG g; memset(&g, 0, sizeof g);
    g.in = c.in; g.wp = c.wp; g.ldw = c.ldw; g.bias = c.bias; g.rowvec = c.rowvec; g.rowvec_ld = c.rowvec_ld;
    g.residual = c.residual; g.out = c.out; g.out_nchw_f32 = 0;
    g.B = c.B; g.Hi = c.Hi; g.Wi = c.Wi; g.Ho = c.Ho; g.Wo = c.Wo; g.Co = c.Co; g.ksize = c.ksize; g.stride = c.stride;
    g.pad = (c.map == MAP_NORMAL && c.stride == 1) ? c.ksize / 2 : 0; g.map = c.map; g.accumulate = c.accumulate ? 1 : 0;
    const dim3 grid((unsigned)((Pout + 63) / 64), (unsigned)((c.Co + 63) / 64));
    S.push_back({"[simt]", fl, ATTN_STEP_SIMT, 1, [g, grid](cudaStream_t st) { launch_k(k_conv_generic, grid, 256, 0, st, g); return (int)cudaGetLastError(); }});
    if (c.has_skip) {
        ConvG s = g; s.in = c.skip; s.wp = c.wp + (long long)taps * Cin; s.ksize = 1; s.pad = 0; s.map = MAP_NORMAL; s.stride = 1;
        s.bias = nullptr; s.rowvec = nullptr; s.residual = nullptr; s.accumulate = 1;
        S.push_back({".skip[simt]", 0, ATTN_STEP_AUX, 1, [s, grid](cudaStream_t st) { launch_k(k_conv_generic, grid, 256, 0, st, s); return (int)cudaGetLastError(); }});
    }
    return 0;
}

// Data gradient of the stride-2 conv (down_conv) on the tensor cores: four output-parity sub-convolutions over dY (4 + 2 + 2 + 1
// taps) whose epilogues scatter to the (2y+py, 2x+px) pixels of dx [B][h][w][C], reading the PK_CONV dkind-3 pack [C][9C]
// (accumulate: dx += as a residual read of dx itself)
inline bool conv_s2_dgrad_tc(int C, int h, int w) { return (C % 64 == 0) && conv_tc_geom(h / 2, w / 2); }
inline int conv_s2_dgrad_steps(ConvSteps& S, const bf16* dY, int B, int h, int w, int C, const bf16* wd, long long ld_d, bf16* dx, bool accumulate, bool dry) {
    const double fl = 2.0 * ((long long)B * (h / 2) * (w / 2)) * C * 9.0 * C;
    int q = 0;
    for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px, ++q) {
        ddpm_gemm_desc d; memset(&d, 0, sizeof d);
        d.mode = GEMM_KK; d.M = B * (h / 2) * (w / 2); d.N = C; d.W = w / 2; d.H = h / 2; d.NB = B;
        d.a_ptr[0] = dY; d.a_C[0] = C; d.a_ld[0] = C;
        d.nseg = 1; d.seg_map[0] = 0; d.seg_kchunks[0] = C / 64; d.seg_cbase[0] = 0; d.seg_custom[0] = 1; d.seg_cmul[0] = 1;
        int nt = 0;
        for (int ky = py ? 1 : 0; ky < 3; ky += 2) for (int kx = px ? 1 : 0; kx < 3; kx += 2) {
            d.seg_dy[0][nt] = (signed char)(-(ky / 2)); d.seg_dx[0][nt] = (signed char)(-(kx / 2)); ++nt;
            if (px) break;
        }
        // (the loops above enumerate ky in {0,2} or {1} and kx in {0,2} or {1}, kx fastest)
        d.seg_taps[0] = nt;
        d.b_ptr = wd; d.b_K = 9 * C; d.b_rows = C; d.b_batch = 1; d.b_ld = ld_d;
        d.b_k_base = (py == 0 ? (px == 0 ? 0 : 4) : (px == 0 ? 6 : 8)) * C;
        d.out = dx; d.ldo = C; d.alpha = 1.f; d.grid_z = 1; d.o_mul = 2; d.o_py = py; d.o_px = px;
        if (accumulate) { d.residual = dx; d.ldr = C; }
        if (dry) { S.push_back({"", q ? 0 : fl, ATTN_STEP_TC, 1, [](cudaStream_t) { return 0; }}); continue; }
        GemmLaunch g; const int rc = build_gemm(d, g);
        if (rc) return rc;
        S.push_back({"", q ? 0 : fl, ATTN_STEP_TC, 1, [g](cudaStream_t st) { return launch_gemm(g, st); }});
    }
    return 0;
}

// Nearest-2x upsample + 3x3 conv (unet.py:199-202) with the upsampled tensor never materialised: four output-parity
// sub-convolutions with 2x2 taps over the low-resolution x [B][h][w][C] (merged weights, PK_UPFOLD [C][16C]) scatter to the
// (2y+py, 2x+px) pixels of out [B][2h][2w][C]: 4/9 of the MACs, no 2x copy.  qstats: the output's quad statistics (or null).
inline bool conv_fold_ok(int C, int h, int w) { return C % 256 == 0 && conv_tc_geom(h, w); }
inline int conv_fold_steps(ConvSteps& S, const bf16* x, int B, int h, int w, int C, const bf16* wf, long long ld_f, const float* bias,
                           bf16* out, double* qstats, bool dry) {
    const double fl = 2.0 * ((long long)B * 4 * h * w) * C * 9.0 * C;       // the reference's count (the folded form does 4/9 of it)
    for (int q = 0; q < 4; ++q) {
        const int py = q >> 1, px = q & 1;
        ddpm_gemm_desc d; memset(&d, 0, sizeof d);
        d.mode = GEMM_KK; d.M = B * h * w; d.N = C; d.W = w; d.H = h; d.NB = B;
        d.a_ptr[0] = x; d.a_C[0] = C; d.a_ld[0] = C;
        d.nseg = 1; d.seg_map[0] = 0; d.seg_kchunks[0] = C / 64; d.seg_cbase[0] = 0; d.seg_custom[0] = 1; d.seg_cmul[0] = 1; d.seg_taps[0] = 4;
        for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) {
            d.seg_dy[0][a * 2 + b] = (signed char)(py == 0 ? a - 1 : a); d.seg_dx[0][a * 2 + b] = (signed char)(px == 0 ? b - 1 : b);
        }
        d.b_ptr = wf; d.b_K = 16 * C; d.b_rows = C; d.b_batch = 1; d.b_ld = ld_f; d.b_k_base = q * 4 * C;
        d.out = out; d.ldo = C; d.alpha = 1.f; d.grid_z = 1; d.o_mul = 2; d.o_py = py; d.o_px = px;
        d.bias = bias; d.gn.qstats = qstats;
        if (dry) { S.push_back({"[fold]", q ? 0 : fl, ATTN_STEP_TC, 1, [](cudaStream_t) { return 0; }}); continue; }
        GemmLaunch g; const int rc = build_gemm(d, g);
        if (rc) return rc;
        S.push_back({"[fold]", q ? 0 : fl, ATTN_STEP_TC, 1, [g](cudaStream_t st) { return launch_gemm(g, st); }});
    }
    return 0;
}

// weight gradient dW (OIHW fp32) of a conv from dy [B][Ho][Wo][Co] and the conv input `in` on an Hi x Wi map
struct WgradArgs {
    const bf16* dy = nullptr; int B = 0, Ho = 0, Wo = 0, Co = 0, Co_valid = 0;
    GnSrc in{}; int Hi = 0, Wi = 0;
    int ksize = 3, stride = 1, map = MAP_NORMAL;
    float* dw = nullptr;
    int Cin() const { return in.C0 + in.C1; }
};
inline bool wgrad_s2(const WgradArgs& w) { return w.stride == 2 && w.ksize == 3 && w.in.C1 == 0 && w.Hi == 2 * w.Ho && w.Wi == 2 * w.Wo; }
inline bool wgrad_route_tc(const WgradArgs& w) {
    const bool s2 = wgrad_s2(w);
    return (w.stride == 1 || s2) && w.map == MAP_NORMAL && w.Co % 64 == 0 && w.Co == w.Co_valid && w.in.C0 % 64 == 0 && w.in.C1 % 64 == 0 &&
           conv_tc_geom(w.Ho, w.Wo) && (s2 || w.Hi == w.Ho);
}
// split count of source s of a tensor-core weight gradient: ONE full wave (<= kPlanSms CTAs), since more splits only add epilogue
// atomics and kPlanSms*k + 1 CTAs would cost a whole extra wave (1x1 weight gradients are a few output tiles and HBM-bound: half a
// wave leaves the other SMs to the main chain)
inline int wgrad_splits(const WgradArgs& w, int Cs, int* block_n) {
    const int taps = w.ksize * w.ksize, kblocks = (int)(((long long)w.B * w.Ho * w.Wo + 63) / 64);
    const int bn = pick_block_n(Cs);
    const int tiles = ((w.Co + 127) / 128) * (Cs / bn) * taps;
    int splits = ((taps == 1 && tiles <= 12) ? kPlanSms / 2 : kPlanSms) / tiles; if (splits > kblocks / 4) splits = kblocks / 4; if (splits < 1) splits = 1;
    if (block_n) *block_n = bn;
    return splits;
}
// Tensor-core route: one MNMN GEMM per concat source (fp32 atomics: 1x1 into dw, which must hold zeros or the sum so far; 3x3 into
// scratch9 = zeroed [9][Co][Cin], after which *unpack, a PK_UNPACK_GRAD row, writes dw and clears the scratch).
// CUDA cores: k_wgrad_generic, accumulating into dw.
inline int wgrad_steps(ConvSteps& S, const WgradArgs& w, float* scratch9, PackEntry* unpack, bool dry) {
    const int Cin = w.Cin(), taps = w.ksize * w.ksize, Co = w.Co;
    const long long P = (long long)w.B * w.Ho * w.Wo;
    const double fl = 2.0 * P * w.Co_valid * (double)taps * Cin;
    if (wgrad_route_tc(w)) {
        const bool s2 = wgrad_s2(w);
        if (taps == 9 && !scratch9 && !dry) return fail(-31, "internal: 3x3 weight gradient without its scratch");
        for (int s = 0; s < (w.in.C1 ? 2 : 1); ++s) {
            const bf16* a = s ? w.in.x1 : w.in.x0; const int Cs = s ? w.in.C1 : w.in.C0, coff = s ? w.in.C0 : 0;
            ddpm_gemm_desc d; memset(&d, 0, sizeof d);
            d.mode = GEMM_MNMN; d.M = Co; d.N = Cs; d.W = w.Wo; d.H = w.Ho; d.NB = w.B;
            d.a_ptr[0] = w.dy; d.a_C[0] = Co; d.a_ld[0] = Co;
            d.b_ptr = a; d.b_K = Cs; d.b_ld = Cs;
            if (s2) { d.b_estride = 2; d.b_pad = 0; }
            d.taps = taps; d.kblocks = (int)((P + 63) / 64);
            d.splits = wgrad_splits(w, Cs, nullptr); d.grid_z = taps * d.splits;
            d.flags = EPI_OUT_F32 | EPI_ATOMIC; d.alpha = 1.f;
            if (taps == 9) { d.out = scratch9 + coff; d.ldo = Cin; d.out_tap_stride = (long long)Co * Cin; }
            else { d.out = w.dw + coff; d.ldo = Cin; }
            if (dry) { S.push_back({"", s ? 0 : fl, ATTN_STEP_TC, 1, [](cudaStream_t) { return 0; }}); continue; }
            GemmLaunch g; const int rc = build_gemm(d, g);
            if (rc) return rc;
            S.push_back({"", s ? 0 : fl, ATTN_STEP_TC, 1, [g](cudaStream_t st) { return launch_gemm(g, st); }});
        }
        if (taps == 9 && unpack) *unpack = unpack_grad_entry(scratch9, w.dw, Co, Cin);
        return 0;
    }
    WgradG g; memset(&g, 0, sizeof g);
    g.dy = w.dy; g.in = w.in; g.dw = w.dw; g.s_co = (long long)Cin * taps; g.s_ci = taps; g.s_tap = 1;
    g.B = w.B; g.Hi = w.Hi; g.Wi = w.Wi; g.Ho = w.Ho; g.Wo = w.Wo; g.Co = Co; g.ksize = w.ksize; g.stride = w.stride;
    g.pad = (w.map == MAP_NORMAL && w.stride == 1) ? w.ksize / 2 : 0; g.map = w.map; g.Co_valid = w.Co_valid;
    const int tiles = ((Cin + 63) / 64) * ((Co + 63) / 64) * taps;
    int splits = (592 + tiles - 1) / tiles; const int maxs = (int)((P + 255) / 256); if (splits > maxs) splits = maxs; if (splits < 1) splits = 1;
    g.pix_per_split = (int)(((P + splits - 1) / splits + 15) / 16 * 16);
    splits = (int)((P + g.pix_per_split - 1) / g.pix_per_split);
    const dim3 grid((Cin + 63) / 64, (Co + 63) / 64, taps * splits);
    S.push_back({"[simt]", fl, ATTN_STEP_SIMT, 1, [g, grid](cudaStream_t st) { launch_k(k_wgrad_generic, grid, 256, 0, st, g); return (int)cudaGetLastError(); }});
    return 0;
}

struct UnetEngine {
    ddpm_unet_cfg cfg;
    bool resample_with_conv = true;       // false: AvgPool2d(2) / bare nearest x2 instead of the resample convs (unet.py:164-170,199-202)
    std::vector<ParamInfo> params;
    std::map<std::string, int> pidx;
    long long flat_elems = 0;
    // bound buffers
    float* P = nullptr; float* G = nullptr;
    uint8_t* ws = nullptr; size_t ws_bytes = 0;
    // plan state
    int B = 0, H = 0, W = 0; bool train = false; bool dry = true; size_t cursor = 0; bool planned = false;
    std::vector<Op> pack_ops, fwd_ops, bwd_ops;
    size_t first_packed_op = 0;
    std::vector<std::function<void()>> tape;
    std::vector<std::string> tape_tag; std::string cur_tag = "late";       // gradient-chunk group of every tape entry
    void tape_push(std::function<void()> f) { tape.push_back(std::move(f)); tape_tag.push_back(cur_tag); }
    std::vector<GradChunk> chunks;
    std::map<long long, std::pair<T4, bool>> grads;     // fwd tensor offset -> (grad tensor, written?)
    size_t zero_fwd_off = 0, zero_fwd_bytes = 0, zero_bwd_off = 0, zero_bwd_bytes = 0;   // per-pass zeroed regions
    size_t once_zero_off = 0, once_zero_bytes = 0;                                       // zeroed at plan time only
    std::vector<SgemmParams> tp_table_host; size_t tp_table_off = 0; int tp_max_c = 0;
    std::vector<SgemmParams> tp_uni_table_host; size_t tp_uni_table_off = 0;
    std::vector<Op> temb_uni_ops;          // one-row timestep path + broadcast (sampler: the whole batch shares t)
    std::vector<FcEnt> fc_table_host; size_t fc_table_off = 0;   // tensor-core timestep projections (concatenated fc weights)
    bool uniform_t = false;                // set by ddpm_sampler_step around its forward
    std::vector<SgemmParams> tpw_table_host, tpd_table_host; size_t tpw_table_off = 0, tpd_table_off = 0;
    // the timestep path's buffers and layout as planned (read by the ddpm_unet_temb_* probes); block names in tp_entry order
    struct TembBufs { float *emb = nullptr, *e0 = nullptr, *e1 = nullptr, *TP = nullptr, *dTP = nullptr, *d_st = nullptr, *d_s0 = nullptr;
                      int E = 0, tp_ld = 0, maxc = 0; bool tc = false; } temb;
    std::vector<std::string> tp_block_host;
    // the image-side convolutions as planned (read by the ddpm_unet_image_* probes): routes 1 = tensor cores, 0 = CUDA cores,
    // -1 = not in this plan (weight gradient and dx of an inference plan); h0 and its quad statistics, out_conv.0's output a,
    // and the gradients d_a (of a) and dh0 (of h0)
    struct ImgBufs { int in_tc = -1, in_wgrad_tc = -1, out_tc = -1, dx_tc = -1;
                     bf16 *h0 = nullptr, *a = nullptr, *d_a = nullptr, *dh0 = nullptr; double* h0_qs = nullptr; } img;
    uint32_t layer_counter = 0;
    double fwd_flops = 0, bwd_flops = 0;
    int n_tc_gemms = 0, n_generic = 0;
    // per-call IO (read by ops at run time)
    const float* x_in = nullptr; const long long* t_in = nullptr; float* eps_out = nullptr;
    unsigned long long drop_seed = 0;
    // backward variant of the current run (ddpm_unet_backward_ex): the ops run per Op::runs(bwd_dx, bwd_params)
    bool bwd_params = true, bwd_dx = false;
    float* dx_dst = nullptr;               // dx f32 [B, Cin, H, W] NCHW of the input-gradient op
    bool chunks_current = true;            // false after a backward without parameter gradients: no chunk event was recorded
    float* out_T = nullptr;                // [P][32] tap outputs of the tensor-core out_conv (forward only; reused by the dx op)
    float* gn_sink = nullptr;              // [2][kGnMaxC] GroupNorm dgamma / dbeta target of a backward without parameter gradients
                                           // (accumulated into, never read)
    // diffusion-side internal buffers
    size_t xt_off = 0, eps_off = 0, tbuf_off = 0, coefcur_off = 0, counter_off = 0, deps_off = 0;
    size_t bpd_part_off = 0;               // bits/dim per-block partial sums [B * ceil(H*W/256)][2]

    // ------------------------------------------------------------------ parameters (reference registration order)
    void add_param(const std::string& n, std::initializer_list<int> d) {
        ParamInfo p; p.name = n; p.nd = (int)d.size(); p.numel = 1; int i = 0;
        for (int v : d) { p.dims[i++] = v; p.numel *= v; }
        for (; i < 4; ++i) p.dims[i] = 1;
        p.off = flat_elems; flat_elems += (p.numel + 63) / 64 * 64;
        pidx[n] = (int)params.size(); params.push_back(p);
    }
    void reg_lin(const std::string& p, int i, int o) { add_param(p + ".weight", {o, i}); add_param(p + ".bias", {o}); }
    void reg_conv(const std::string& p, int i, int o, int k) { add_param(p + ".weight", {o, i, k, k}); add_param(p + ".bias", {o}); }
    void reg_gn(const std::string& p, int n) { add_param(p + ".weight", {n}); add_param(p + ".bias", {n}); }
    void reg_res(const std::string& p, int i, int o) {
        reg_gn(p + ".norm1", i); reg_conv(p + ".conv1", i, o, 3); reg_lin(p + ".fc", cfg.temb_dim, o);
        reg_gn(p + ".norm2", o); reg_conv(p + ".conv2", o, o, 3);
        if (i != o) reg_conv(p + ".skip", i, o, 1);
    }
    void reg_attn(const std::string& p, int n) { reg_gn(p + ".norm", n); reg_conv(p + ".project_in", n, 3 * n, 1); reg_conv(p + ".project_out", n, n, 1); }
    void reg_block(const std::string& p, int i, int o, bool at) { if (at) { reg_res(p + ".0", i, o); reg_attn(p + ".1", o); } else reg_res(p, i, o); }
    int chs(int l) const { return cfg.hid_channels * cfg.ch_mult[l]; }
    void register_params() {
        const int ch = cfg.hid_channels, L = cfg.levels, nrb = cfg.num_res_blocks, E = cfg.temb_dim;
        reg_lin("embed.0", ch, E); reg_lin("embed.2", E, E);
        reg_conv("in_conv", cfg.in_channels, ch, 3);
        for (int i = 0; i < L; ++i) {
            const int prev = i ? chs(i - 1) : ch, cur = chs(i);
            const std::string p = "downsamples.level_" + std::to_string(i);
            reg_block(p + ".0", prev, cur, cfg.attn[i]);
            for (int j = 1; j < nrb; ++j) reg_block(p + "." + std::to_string(j), cur, cur, cfg.attn[i]);
            if (i != L - 1 && resample_with_conv) reg_conv(p + "." + std::to_string(nrb) + ".1", cur, cur, 3);
        }
        const int mid = chs(L - 1);
        reg_res("middle.0", mid, mid); reg_attn("middle.1", mid); reg_res("middle.2", mid, mid);
        for (int i = 0; i < L; ++i) {
            const int nxt = i == 0 ? ch : chs(i - 1), prev = i == L - 1 ? chs(L - 1) : chs(i + 1), cur = chs(i);
            const std::string p = "upsamples.level_" + std::to_string(i);
            reg_block(p + ".0", prev + cur, cur, cfg.attn[i]);
            for (int j = 1; j < nrb; ++j) reg_block(p + "." + std::to_string(j), 2 * cur, cur, cfg.attn[i]);
            reg_block(p + "." + std::to_string(nrb), nxt + cur, cur, cfg.attn[i]);
            if (i != 0 && resample_with_conv) reg_conv(p + "." + std::to_string(nrb + 1) + ".1", cur, cur, 3);
        }
        reg_gn("out_conv.0", ch); reg_conv("out_conv.2", ch, cfg.out_channels, 3);
        layout_params();
    }
    // Memory layout of the flat buffers: registration order, EXCEPT that the tensors whose gradients only exist at the very end
    // of the backward pass (the embedding MLP and the per-block timestep projections fc.weight, unet.py:122-126,77) are moved
    // behind everything else ("late region"), so that the rest forms contiguous per-level ranges that complete one after the
    // other.  The parameter LIST (state_dict order) is unchanged - only the offsets differ.
    static bool is_late(const std::string& n) { return n.rfind("embed.", 0) == 0 || (n.size() > 10 && n.compare(n.size() - 10, 10, ".fc.weight") == 0); }
    long long main_elems = 0;
    void layout_params() {
        long long off = 0;
        for (auto& p : params) if (!is_late(p.name)) { p.off = off; off += (p.numel + 63) / 64 * 64; }
        main_elems = off;
        for (auto& p : params) if (is_late(p.name)) { p.off = off; off += (p.numel + 63) / 64 * 64; }
        flat_elems = off;
    }
    // group of a parameter / tape entry for the gradient chunks: d<i> (in_conv + down level i), mid, u<i> (+ out_conv), late
    std::string group_of(const std::string& n) const {
        if (is_late(n)) return "late";
        if (n.rfind("in_conv", 0) == 0) return "d0";
        if (n.rfind("out_conv", 0) == 0) return "u" + std::to_string(cfg.levels - 1);
        if (n.rfind("middle", 0) == 0) return "mid";
        const size_t k = n.find("level_");
        if (k != std::string::npos) return std::string(n[0] == 'd' ? "d" : "u") + std::to_string(atoi(n.c_str() + k + 6));
        return "late";
    }
    const ParamInfo& pinfo(const std::string& n) const { return params[pidx.at(n)]; }
    float* PP(const std::string& n) const { return P + pinfo(n).off; }
    float* GP(const std::string& n) const { return G ? G + pinfo(n).off : nullptr; }

    // ------------------------------------------------------------------ workspace
    size_t alloc(size_t bytes) { const size_t o = (cursor + 1023) & ~size_t(1023); cursor = o + bytes; return o; }
    template <class T> T* at(size_t off) const { return reinterpret_cast<T*>(ws + off); }
    T4 newT(int b, int h, int w, int c) { T4 t; t.B = b; t.H = h; t.W = w; t.C = c; t.off = (long long)alloc((size_t)t.numel() * 2); return t; }
    bf16* bp(const T4& t) const { return at<bf16>((size_t)t.off); }
    GnSrc gsrc(const Src& s) const { GnSrc g; g.x0 = bp(s.t0); g.C0 = s.t0.C; g.x1 = s.two ? bp(s.t1) : nullptr; g.C1 = s.two ? s.t1.C : 0; return g; }
    static Src one(const T4& t) { Src s; s.t0 = t; s.two = false; return s; }

    // role given to backward ops as they are pushed (RoleScope sets it around a builder)
    int push_role = ROLE_DATA;
    struct RoleScope { UnetEngine* e; int prev; RoleScope(UnetEngine* e_, int r) : e(e_), prev(e_->push_role) { e->push_role = r; } ~RoleScope() { e->push_role = prev; } };
    void push(std::vector<Op>& L, const std::string& name, double flops, std::function<int(cudaStream_t)> f, int launches = 1, bool side = false) {
        Op o; o.name = name; o.flops = flops; o.run = std::move(f); o.launches = launches; o.side = side;
        if (&L == &bwd_ops) o.role = push_role;
        L.push_back(std::move(o));
    }
    static int count_launches(const std::vector<Op>& L) { int n = 0; for (auto& o : L) n += o.launches; return n; }
    int count_bwd_launches(bool want_dx, bool param_grads) const { int n = 0; for (auto& o : bwd_ops) if (o.runs(want_dx, param_grads)) n += o.launches; return n; }
    // grad tensor of a forward tensor; `first` tells the producer whether to overwrite (=) or accumulate (+=)
    T4 grad_of(const T4& t, bool* first) {
        auto it = grads.find(t.off);
        if (it == grads.end()) { T4 g = newT(t.B, t.H, t.W, t.C); it = grads.emplace(t.off, std::make_pair(g, false)).first; }
        if (first) { *first = !it->second.second; it->second.second = true; }
        return it->second.first;
    }
    bool has_grad(const T4& t) const { auto it = grads.find(t.off); return it != grads.end() && it->second.second; }

    // ------------------------------------------------------------------ op builders
    bool tc_ok_geom(int h, int w) const { return conv_tc_geom(h, w); }

    // conv: out = conv(in) [+ 1x1 skip(skip_in)] + bias + rowvec[b] + residual ; packed weights [Co][ldw]
    struct ConvSpec {
        std::string name; Src in; int ksize = 3, stride = 1, map = MAP_NORMAL;
        const bf16* wp = nullptr; long long ldw = 0; bool has_skip = false; Src skip_in;
        bool skip_identity = false;        // the skip chunks carry identity weights (the block's residual): no FLOPs of the reference's count
        const float* bias = nullptr; const float* rowvec = nullptr; int rowvec_ld = 0; const bf16* residual = nullptr;
        T4 out; int Co = 0; int Ho = 0, Wo = 0; bool accumulate = false;
        bool want_qstats = false;          // the output feeds a GroupNorm -> statistics in the epilogue when the kernel can
        const float* xfK = nullptr; int xf_silu = 0;   // inference: `in` is the RAW GroupNorm input, the conv applies act(sc*x + sh) in its
                                                       // operand path (haloed kernel only; see xf_ok / gn_prep_xf)
    };
    // GroupNorm(+SiLU) folded into the consumer 3x3 conv's operand path (conv_halo.cuh, xfK): inference plans, single-source input with
    // producer statistics, and a conv that takes the haloed kernel.
    // OPT-IN (DDPM_XF=1, read at plan time): the rewrite of the landed tile serialises with the conv's MMAs, against the apply pass
    // (read x + write a) it removes; not measured on H100.  Kept, with unit and network parity tests.
    bool xf_ok(const Src& x, int Co, int h, int w) const {
        const char* on = getenv("DDPM_XF");
        const bool off = !on || atoi(on) == 0 || getenv("DDPM_NO_GN_EPI") != nullptr || getenv("DDPM_NO_HALO") != nullptr;
        if (off || train || x.two || x.t0.qs < 0 || x.t0.C % 128 || Co % 128) return false;
        return halo_eligible(h, w, Co) && tc_ok_geom(h, w);
    }
    float* gn_prep_xf(std::vector<Op>& L, const std::string& name, const Src& in, const std::string& pname) {
        const int C = in.C(), Bn = in.t0.B, HW = in.t0.H * in.t0.W;
        gn_check(name, C);
        float* K = at<float>(alloc((size_t)Bn * 4 * C * 4));
        GnApply a; memset(&a, 0, sizeof a);
        a.s = gsrc(in); a.HW = HW; a.qs0 = at<double>((size_t)in.t0.qs); a.qs1 = nullptr;
        a.gamma = PP(pname + ".weight"); a.beta = PP(pname + ".bias"); a.eps = 1e-6f; a.Kout = K;
        push(L, name + ".prep", 0, [a, Bn](cudaStream_t st) { return launch_gn_prep(a, Bn, st); });
        return K;
    }
    // epilogue fusion of a conv: fills `gn` and returns the workspace offset of the quad statistics (-1: none)
    long long conv_gn_epi(const ConvSpec& c, ddpm_gn_epi& gn) {
        memset(&gn, 0, sizeof gn);
        long long qs = -1;
        static const bool no_fuse = getenv("DDPM_NO_GN_EPI") != nullptr;
        if (no_fuse) return qs;
        const int Bn = c.in.t0.B, HW = c.Ho * c.Wo;
        if (c.want_qstats && c.Co % 32 == 0 && HW % 32 == 0) {
            qs = (long long)zero_fwd((size_t)Bn * (c.Co / 4) * 2 * 8);
            gn.qstats = at<double>((size_t)qs);
        }
        return qs;
    }
    // the launch steps of a conv builder as ops named name + step.name; side: forked onto the side stream
    void push_conv_steps(std::vector<Op>& L, const std::string& name, const ConvSteps& steps, double* flops_acc, bool side = false) {
        for (const ConvStep& s : steps) {
            if (flops_acc) *flops_acc += s.flops;
            if (s.kind == ATTN_STEP_TC) ++n_tc_gemms;
            else if (s.kind == ATTN_STEP_SIMT) ++n_generic;
            push(L, name + s.name, s.flops, s.run, s.launches, side);
        }
    }
    long long conv_op(std::vector<Op>& L, const ConvSpec& c, double* flops_acc) {
        ConvArgs a;
        a.in = gsrc(c.in); a.B = c.in.t0.B; a.Hi = c.in.t0.H; a.Wi = c.in.t0.W; a.ksize = c.ksize; a.stride = c.stride; a.map = c.map;
        a.wp = c.wp; a.ldw = c.ldw; a.has_skip = c.has_skip; a.skip_identity = c.skip_identity;
        if (c.has_skip) a.skip = gsrc(c.skip_in);
        a.bias = c.bias; a.rowvec = c.rowvec; a.rowvec_ld = c.rowvec_ld; a.residual = c.residual;
        a.out = bp(c.out); a.Co = c.Co; a.Ho = c.Ho; a.Wo = c.Wo; a.accumulate = c.accumulate; a.xfK = c.xfK; a.xf_silu = c.xf_silu;
        static const bool no_halo = getenv("DDPM_NO_HALO") != nullptr;
        static const bool no_n128 = getenv("DDPM_NO_N128_FILL") != nullptr;
        const ConvChoice ch = conv_choose(a, !no_halo, !no_n128);
        if (c.xfK && ch.route != CONV_ROUTE_HALO) { plan_error = fail(-31, "internal: conv '%s' was planned with a fused GroupNorm input but did not take the haloed kernel", c.name.c_str()); return -1; }
        long long qs = -1; float* scratch = nullptr;
        if (ch.splits > 1) scratch = at<float>(alloc_once_zero((size_t)a.B * c.Ho * c.Wo * c.Co * 4));
        else if (ch.route != CONV_ROUTE_SIMT) { ddpm_gn_epi gn; qs = conv_gn_epi(c, gn); a.qstats = gn.qstats; }
        ConvSteps steps;
        const int rc = conv_fwd_steps(steps, a, ch, scratch, dry);
        if (rc) { plan_error = rc; return qs; }
        push_conv_steps(L, c.name, steps, flops_acc);
        return qs;
    }
    float* eps_dst = nullptr;   // run-time destination of the final conv (caller buffer or internal eps buffer)
    PsampleEpi ps_epi = {nullptr, nullptr, nullptr, 0, nullptr};   // run-time: sampler update fused into the final gather (x != null)
    QsamplePro qs_pro = {};           // run-time: q_sample fused into in_conv's loads (ddpm_train_forward, ddpm_bpd_step)
    BpdEpi bpd_epi = {};              // run-time: bits/dim terms fused into the final gather (part != null; ddpm_bpd_step)
    bool gather_fused_tail = false;   // plan property: the final conv ends in k_out_gather (tensor-core out_conv path)
    const float* deps_src = nullptr;   // run-time d(loss)/d(eps), fp32 NCHW (caller buffer or internal buffer)
    int plan_error = 0;

    // weight gradient of a conv: dW (OIHW fp32, flat grads) from dy [B,Ho,Wo,Co] and the conv input
    void wgrad_op(const std::string& name, const T4& dy, const Src& in, int ksize, int stride, int map, float* dw, int Co_valid) {
        RoleScope role(this, ROLE_PARAM);
        WgradArgs w;
        w.dy = bp(dy); w.B = dy.B; w.Ho = dy.H; w.Wo = dy.W; w.Co = dy.C; w.Co_valid = Co_valid;
        w.in = gsrc(in); w.Hi = in.t0.H; w.Wi = in.t0.W; w.ksize = ksize; w.stride = stride; w.map = map; w.dw = dw;
        const bool tc = wgrad_route_tc(w);
        // 3x3 on the tensor cores: packed [tap][Co][Ci] scratch -> OIHW flat gradient, batched into ONE table-driven launch at the
        // end of backward
        float* scratch = (tc && ksize == 3) ? at<float>(alloc_once_zero((size_t)9 * w.Co * w.Cin() * 4)) : nullptr;
        ConvSteps steps; PackEntry unpack;
        const int rc = wgrad_steps(steps, w, scratch, &unpack, dry);
        if (rc) { plan_error = rc; return; }
        // weight gradients are leaves of the backward graph: run them on the side stream, where the tensor-bound GEMMs
        // overlap the memory-bound GroupNorm kernels of the main chain (DDPM_WGRAD_MAIN=1 keeps the tensor-core ones in line)
        static const bool wg_side = getenv("DDPM_WGRAD_MAIN") == nullptr;
        push_conv_steps(bwd_ops, name, steps, &bwd_flops, tc ? wg_side : true);
        if (scratch) unpack_table_host.push_back(unpack);
    }
    size_t alloc_once_zero(size_t bytes) {   // carve from the plan-time-zeroed arena (contiguous region grown on demand)
        const size_t o = alloc(bytes);
        once_list.push_back({o, bytes});
        return o;
    }
    std::vector<std::pair<size_t, size_t>> once_list;

    // per-pass zeroed arenas (GroupNorm statistic accumulators etc.): bump-allocated inside a region zeroed by ONE memset
    size_t zf_cursor = 0, zb_cursor = 0;
    size_t zero_fwd(size_t bytes) { const size_t o = zf_cursor; zf_cursor += (bytes + 255) & ~size_t(255); return zero_fwd_off + o; }
    size_t zero_bwd(size_t bytes) { const size_t o = zb_cursor; zb_cursor += (bytes + 255) & ~size_t(255); return zero_bwd_off + o; }

    // a GroupNorm over more than kGnMaxC concat channels has no launch geometry: refuse the plan, naming the first such layer
    void gn_check(const std::string& name, int C) {
        if (C > kGnMaxC && !plan_error)
            plan_error = fail(-30, "GroupNorm '%s' has %d channels; the GroupNorm kernels support at most %d", name.c_str(), C, kGnMaxC);
    }
    GnSaved gn_fwd(std::vector<Op>& L, const std::string& name, const Src& in, const std::string& pname, const T4& out, int silu, float drop_p) {
        const int C = in.C(), Bn = in.t0.B, HW = in.t0.H * in.t0.W;
        gn_check(name, C);
        GnSaved sv; sv.in = in; sv.silu = silu; sv.drop_p = drop_p; sv.layer = ++layer_counter;
        sv.gamma = PP(pname + ".weight"); sv.beta = PP(pname + ".bias"); sv.dgamma = GP(pname + ".weight"); sv.dbeta = GP(pname + ".bias");
        double* stats = at<double>(zero_fwd((size_t)Bn * 64 * 8));
        sv.K = at<float>(alloc((size_t)Bn * 4 * C * 4));
        const GnSrc gs = gsrc(in);
        float* K = sv.K; const float* ga = sv.gamma; const float* be = sv.beta;
        sv.mask = (drop_p > 0.f && train) ? at<unsigned char>(alloc((size_t)Bn * HW * (C / 8))) : nullptr;
        GnApply a; memset(&a, 0, sizeof a);
        a.s = gs; a.K = K; a.y = bp(out); a.HW = HW; a.silu = silu; a.drop_p = sv.drop_p; a.seed = 0; a.layer = sv.layer; a.mask = sv.mask;
        UnetEngine* self = this;
        // statistics delivered by the producers' epilogues (conv_gn_epi): one launch, no pass over the tensor for the stats
        const bool have_qs = in.t0.qs >= 0 && (!in.two || in.t1.qs >= 0) && (C % 128) == 0;
        if (have_qs) {
            a.qs0 = at<double>((size_t)in.t0.qs); a.qs1 = in.two ? at<double>((size_t)in.t1.qs) : nullptr;
            a.gamma = ga; a.beta = be; a.eps = 1e-6f; a.Kout = K;
            push(L, name + ".apply[qs]", 0, [a, Bn, self](cudaStream_t st) { GnApply aa = a; gn_arm_dropout(aa.drop_p, aa.seed, self->drop_seed);
                return launch_gn_apply(aa, Bn, st); });
            return sv;
        }
        if (HW <= 64 && !getenv("DDPM_NO_GN_EPI")) {       // tiny maps: statistics + apply in ONE launch, one block per image
            a.gamma = ga; a.beta = be; a.eps = 1e-6f; a.Kout = K;
            push(L, name + ".small", 0, [a, Bn, self](cudaStream_t st) { GnApply aa = a; gn_arm_dropout(aa.drop_p, aa.seed, self->drop_seed);
                return launch_gn_small(aa, Bn, st); });
            return sv;
        }
        GnFin fin; fin.gamma = ga; fin.beta = be; fin.K = K; fin.eps = 1e-6f; fin.ticket = at<int>(zero_fwd((size_t)Bn * 4));
        push(L, name + ".stats", 0, [=](cudaStream_t st) { return launch_gn_stats(gs, stats, Bn, HW, fin, st); });
        push(L, name + ".apply", 0, [a, Bn, self](cudaStream_t st) { GnApply aa = a; gn_arm_dropout(aa.drop_p, aa.seed, self->drop_seed);
            return launch_gn_apply(aa, Bn, st); });
        return sv;
    }
    // dx(in) (=|+=) gn_bwd(dy) + addend ; dgamma/dbeta (and the optional column sums) accumulate into the flat grads, except in a
    // backward without parameter gradients, which leaves them out
    void gn_bwd(const std::string& name, const GnSaved& sv, const T4& dy, const bf16* addend,
                float* cs_per_img = nullptr, int cs_ld = 0, float* cs_total = nullptr, float* cs_total2 = nullptr) {
        const Src& in = sv.in;
        const int C = in.C(), Bn = in.t0.B, HW = in.t0.H * in.t0.W;
        GnBwd a; memset(&a, 0, sizeof a);
        a.s = gsrc(in); a.dy = bp(dy); a.K = sv.K; a.gamma = sv.gamma;
        a.cs = at<float>(zero_bwd((size_t)Bn * 2 * C * 4)); a.PQ = at<float>(alloc((size_t)Bn * 2 * C * 4));
        a.dgamma = sv.dgamma; a.dbeta = sv.dbeta;
        bool f0 = true, f1 = true;
        const T4 g0 = grad_of(in.t0, &f0); a.dx0 = bp(g0); a.acc0 = f0 ? 0 : 1;
        if (in.two) { const T4 g1 = grad_of(in.t1, &f1); a.dx1 = bp(g1); a.acc1 = f1 ? 0 : 1; }
        a.addend = addend; a.B = Bn; a.HW = HW; a.silu = sv.silu; a.drop_p = sv.drop_p; a.layer = sv.layer; a.mask = sv.mask;
        a.ticket = at<int>(zero_bwd((size_t)Bn * 4));
        static const bool no_dn = getenv("DDPM_GN_NO_DN") != nullptr;
        a.dn_inplace = (sv.silu && !no_dn) ? 1 : 0;
        UnetEngine* self = this;
        RoleScope role(this, ROLE_MIXED);
        push(bwd_ops, name + ".gn_bwd", 0, [=](cudaStream_t st) {
            GnBwd aa = a; gn_arm_dropout(aa.drop_p, aa.seed, self->drop_seed);
            if (!self->bwd_params) {          // dgamma / dbeta go to the plan's sink, the column sums are not formed
                aa.dgamma = self->gn_sink; aa.dbeta = self->gn_sink + kGnMaxC; return launch_gn_bwd(aa, nullptr, 0, nullptr, nullptr, st); }
            return launch_gn_bwd(aa, cs_per_img, cs_ld, cs_total, cs_total2, st); }, 2);
    }
    void colsum_op(const std::string& name, const T4& dy, float* per_img, int ld, float* total, float* total2, int C_valid) {
        RoleScope role(this, ROLE_PARAM);
        const int HW = dy.H * dy.W, C = dy.C, Bn = dy.B;
        const bf16* p = bp(dy);
        push(bwd_ops, name + ".colsum", 0, [=](cudaStream_t st) { return launch_colsum(p, per_img, ld, total, total2, Bn, HW, C, C_valid, st); }, 1, /*side=*/true);
    }

    // ------------------------------------------------------------------ packed weights (table-driven: one launch re-packs everything)
    struct Packed { bf16* fwd = nullptr; long long ld_f = 0; bf16* dgr = nullptr; long long ld_d = 0; };
    std::vector<PackEntry> pack_table_host, unpack_table_host; size_t pack_table_off = 0, unpack_table_off = 0;
    // fwd pack [Co][taps*Ci (+extra)], dgrad pack [Ci][taps*Co] (dkind 1 plain / 2 flipped taps / 3 stride-2 parity blocks)
    Packed pack_conv(const std::string& pname, int Co, int Ci, int ksize, int extra_k, bool flip, bool want_dgrad, int dkind_override = 0) {
        const int taps = ksize * ksize;
        Packed pk; pk.ld_f = (long long)taps * Ci + extra_k;
        pk.fwd = at<bf16>(alloc((size_t)Co * pk.ld_f * 2));
        if (want_dgrad && train) { pk.ld_d = (long long)taps * Co; pk.dgr = at<bf16>(alloc((size_t)Ci * pk.ld_d * 2)); }
        pack_table_host.push_back(pack_conv_entry(PP(pname + ".weight"), Co, Ci, taps, 0, pk.fwd, pk.ld_f, pk.dgr, pk.ld_d,
                                                  dkind_override ? dkind_override : (flip ? 2 : 1)));
        return pk;
    }
    void pack_extra(const std::string& pname, const Packed& into, int k_off, int Co, int Ci, bf16* dgr, long long ld_d) {
        pack_table_host.push_back(pack_conv_entry(PP(pname + ".weight"), Co, Ci, 1, k_off, into.fwd, into.ld_f, dgr, ld_d, 1));
    }
    void pack_identity(const Packed& into, int k_off, int C) { pack_table_host.push_back(pack_identity_entry(into.fwd, into.ld_f, k_off, C)); }
    void pack_bias_add(float* dst, const float* a, const float* b, int n) { pack_table_host.push_back(pack_bias_add_entry(dst, a, b, n)); }

    // ------------------------------------------------------------------ blocks
    T4 res_block(const std::string& p, const Src& x, int cout, int tp_off, int tp_ld, float* TP, float* dTP);
    T4 attn_block(const std::string& p, const T4& x);
    T4 down_conv(const std::string& p, const T4& x);
    T4 up_conv(const std::string& p, const T4& x);
    T4 down_pool(const std::string& p, const T4& x);
    T4 up_nearest(const std::string& p, const T4& x);
    void push_attn_steps(std::vector<Op>& L, const std::string& p, const AttnSteps& steps, double& flops_acc);
    int plan(int B_, int H_, int W_, bool train_, bool dry_);
    int build();
    // Ops flagged `side` (bias-gradient column sums, gradient unpacks: small, memory-bound, nothing downstream needs them
    // before the end of the pass) are forked onto a second stream so they overlap the tensor-core kernels, and joined at
    // the end of the list.  Fork/join are event edges, so the pattern is CUDA-graph capturable.
    cudaStream_t side_stream = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // Weight repack of a TRAINING plan (every step, after the optimizer): issued on the side stream so that it overlaps the ops
    // of the next forward that do not read packed weights (timestep embedding MLP on the fp32 masters, q_sample + in_conv);
    // the forward list waits on ev_pack_fc / ev_pack_all right before the first consumer (Op::wait_pack).
    cudaEvent_t ev_pack_fork = nullptr, ev_pack_fc = nullptr, ev_pack_all = nullptr; bool pack_pending = false;
    int repack(cudaStream_t st) {
        static const bool inline_pack = getenv("DDPM_PACK_INLINE") != nullptr;
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone; cudaStreamIsCapturing(st, &cs);
        if (!train || !side_stream || !ev_pack_all || inline_pack || cs != cudaStreamCaptureStatusNone || getenv("DDPM_DEBUG_SYNC") || getenv("DDPM_NO_SIDE_STREAM"))
            return run_list(pack_ops, st);
        if (cudaEventRecord(ev_pack_fork, st) || cudaStreamWaitEvent(side_stream, ev_pack_fork, 0)) return fail(-20, "repack fork failed");
        for (int pass = 0; pass < 2; ++pass) {        // early packs (in_conv, timestep MLP: Op::wait_pack == 1) first, then the rest
            for (auto& o : pack_ops) {
                if ((o.wait_pack == 1) != (pass == 0)) continue;
                const int rc = o.run(side_stream);
                if (rc) return fail(-20, "op '%s' failed: %s", o.name.c_str(), cudaGetErrorString((cudaError_t)rc));
            }
            if (pass == 0 && cudaEventRecord(ev_pack_fc, side_stream)) return fail(-20, "repack event failed");
        }
        if (cudaEventRecord(ev_pack_all, side_stream)) return fail(-20, "repack event failed");
        pack_pending = true;
        return 0;
    }
    int run_list(std::vector<Op>& L, cudaStream_t caller_st) {
        cudaStream_t st = caller_st;
        static const bool dbg = getenv("DDPM_DEBUG_SYNC") != nullptr;   // serialise + attribute faults to an op (never under graph capture)
        static const bool no_side = getenv("DDPM_NO_SIDE_STREAM") != nullptr;
        bool forked = false;
        // DDPM_OP_TIMING=<file>: CUDA events after every main-stream op (side stream stays concurrent), appended as "name ms" lines
        static const char* timing_path = getenv("DDPM_OP_TIMING");
        std::vector<cudaEvent_t> tev;
        if (timing_path && !dbg) { tev.resize(L.size() + 1); for (auto& e : tev) cudaEventCreate(&e); cudaEventRecord(tev[0], st); }
        size_t oi = 0; int main_since_fork = 0;
        const bool skip_temb = uniform_t && !temb_uni_ops.empty() && &L == &fwd_ops;
        const bool is_bwd = &L == &bwd_ops;
        for (auto& o : L) {
            int rc;
            ++oi;
            if (is_bwd && !o.runs(bwd_dx, bwd_params)) {
                if (!tev.empty()) cudaEventRecord(tev[oi], st);
                continue;
            }
            if (skip_temb && o.tag == OP_TEMB) {
                if (o.name == "temb.sin") for (auto& u : temb_uni_ops) { rc = u.run(st); if (rc) return fail(-20, "op '%s' failed: %s", u.name.c_str(), cudaGetErrorString((cudaError_t)rc)); }
                if (!tev.empty()) cudaEventRecord(tev[oi], st);
                continue;
            }
            if (o.wait_pack && pack_pending) {
                if (cudaStreamWaitEvent(st, o.wait_pack == 1 ? ev_pack_fc : ev_pack_all, 0)) return fail(-20, "repack join failed");
                if (o.wait_pack == 2) pack_pending = false;
            }
            if (o.chunk >= 0) {
                // gradient-chunk boundary: everything the main chain has written so far is joined into the side stream (which
                // carries the weight-gradient GEMMs), the chunk's gradient unpack runs there, then the chunk's event is recorded
                cudaStream_t cs_ = (side_stream && !dbg && !no_side) ? side_stream : st;
                rc = 0;
                if (cs_ != st) { rc = (int)cudaEventRecord(ev_fork, st); if (!rc) rc = (int)cudaStreamWaitEvent(cs_, ev_fork, 0); main_since_fork = 0; forked = true; }
                if (!rc) rc = o.run(cs_);
                if (!rc && chunks[o.chunk].ev) rc = (int)cudaEventRecord(chunks[o.chunk].ev, cs_);
                if (rc) return fail(-20, "op '%s' failed: %s", o.name.c_str(), cudaGetErrorString((cudaError_t)rc));
                if (!tev.empty()) cudaEventRecord(tev[oi], st);
                continue;
            }
            if (o.side && side_stream && !dbg && !no_side) {
                rc = 0;
                if (main_since_fork || !forked) {     // consecutive side ops share one fork edge
                    rc = (int)cudaEventRecord(ev_fork, st);
                    if (!rc) rc = (int)cudaStreamWaitEvent(side_stream, ev_fork, 0);
                    main_since_fork = 0;
                }
                if (!rc) rc = o.run(side_stream);
                forked = true;
            } else {
                rc = o.run(st);
                ++main_since_fork;
            }
            if (!rc && dbg) rc = (int)cudaStreamSynchronize(st);
            if (rc) return fail(-20, "op '%s' failed: %s", o.name.c_str(), cudaGetErrorString((cudaError_t)rc));
            if (!tev.empty()) cudaEventRecord(tev[oi], st);
        }
        if (forked) {
            int rc = (int)cudaEventRecord(ev_join, side_stream);
            if (!rc) rc = (int)cudaStreamWaitEvent(st, ev_join, 0);
            if (rc) return fail(-20, "side-stream join failed: %s", cudaGetErrorString((cudaError_t)rc));
        }
        if (!tev.empty()) {
            cudaEvent_t fin; cudaEventCreate(&fin); cudaEventRecord(fin, st); cudaStreamSynchronize(st);
            if (FILE* f = fopen(timing_path, "a")) {
                for (size_t i = 0; i < L.size(); ++i) { float ms = 0; cudaEventElapsedTime(&ms, tev[i], tev[i + 1]); fprintf(f, "%s%s %.5f\n", L[i].side ? "[side]" : "", L[i].name.c_str(), ms); }
                float ms = 0; cudaEventElapsedTime(&ms, tev[L.size()], fin); fprintf(f, "[join] %.5f\n", ms);
                fclose(f);
            }
            for (auto& e : tev) cudaEventDestroy(e);
            cudaEventDestroy(fin);
        }
        return 0;
    }
};

}  // namespace ddpm
