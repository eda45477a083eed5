// libddpm_b200.so — single translation unit (device-side error flag and kernels share one module).
#include <cstdarg>
#include <new>
#include <cmath>
#include <climits>
#include <initializer_list>
#include "unet_engine_impl.cuh"
#include "optim.cuh"
#include "knn.cuh"
#include "fid.cuh"
#include "inception.cuh"
#include "inception_score.cuh"
#include "kid.cuh"
#include "toy_mlp.cuh"

using namespace ddpm;

struct ddpm_unet {
    UnetEngine e;
    // sampler tables (device, owned by the handle; allocated by ddpm_sampler_setup, never per step): t_model i64[S], coef f32[S][6]
    void* d_samp = nullptr; int S = 0;
    // bits/dim tables (allocated by ddpm_bpd_setup; separate from the sampler's, whose addresses a captured sampler graph holds):
    // t_model i64[T] = 0..T-1, rows f32[T][kBpdRow], sqrt_ab f32[T], sqrt_1mab f32[T]
    void* d_bpd = nullptr; int bpd_T = 0;
    long long graph_epoch = 0;     // moves whenever an address a captured launch holds may have moved (ddpm_unet_graph_epoch)
    const float* train_target = nullptr;
    bool temb_rows = false;        // the last forward of this plan was a per-row ddpm_unet_temb_forward (what its backward reads);
                                   // every other forward entry point clears it
    bool image_fwd = false;        // the last forward of this plan was a ddpm_unet_image_forward (what its backward reads); cleared likewise
};

__global__ void k_set_int(int* p, int v) {
    pdl_entry(); *p = v; }

extern "C" {

const char* ddpm_last_error(void) { return last_error().c_str(); }

int ddpm_runtime_check(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return fail(-1, "no CUDA device / driver"); }
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceProp pr;
    DDPM_CUDA_OK(cudaGetDeviceProperties(&pr, dev));
    if (pr.major != 9 || pr.minor != 0) return fail(-1, "device %d is sm_%d%d, this library is sm_90a only", dev, pr.major, pr.minor);
    if (!tmap_encode_fn()) return fail(-3, "cuTensorMapEncodeTiled unavailable");
    return 0;
}

int ddpm_device_error_flag(void) {
    unsigned v = 0;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemcpyFromSymbol(&v, g_kernel_error, sizeof v) != cudaSuccess) return -1;
    return (int)v;
}

int ddpm_gemm_run(const ddpm_gemm_desc* d, void* stream) {
    GemmLaunch g;
    int rc = build_gemm(*d, g);
    if (rc) return rc;
    return launch_gemm(g, static_cast<cudaStream_t>(stream));
}

int ddpm_conv_halo_run(const ddpm_halo_desc* d, void* stream) {
    HaloLaunch g;
    int rc = build_halo(*d, g);
    if (rc) return rc;
    return launch_halo(g, static_cast<cudaStream_t>(stream));
}

int ddpm_attn_fused_run(const void* qkv, void* out, void* probs, int NB, int T, int C, void* stream) {
    AttnLaunch g;
    int rc = build_attn(qkv, out, NB, T, C, g, probs);
    if (rc) return rc;
    return launch_attn(g, static_cast<cudaStream_t>(stream));
}

int ddpm_attn_fused_bwd_run(const void* qkv, const void* d_out, const void* probs, void* d_scores, void* d_qkv, int NB, int T, int C, void* stream) {
    AttnLaunch g;
    int rc = build_attn_bwd(qkv, d_out, probs, d_scores, d_qkv, NB, T, C, g);
    if (rc) return rc;
    return launch_attn_bwd(g, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ GroupNorm / column sums
// scratch layout.  forward: stats f64 [B][64] | tickets i32 [B].  backward: cs f32 [B][2][C] | tickets i32 [B] | PQ f32 [B][2][C]
static size_t gn_align(size_t n) { return (n + 255) & ~size_t(255); }
static size_t gn_fwd_scratch(int B) { return gn_align((size_t)B * 64 * 8) + gn_align((size_t)B * 4); }
static size_t gn_bwd_scratch(int B, int C) { return 2 * gn_align((size_t)B * 2 * C * 4) + gn_align((size_t)B * 4); }
static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }
static int gn_check_src(const char* fn, int B, int HW, int C0, int C1, const void* x0, const void* x1) {
    if (B < 1 || HW < 1) return fail(-42, "%s: need B >= 1 and HW >= 1", fn);
    if (C0 < 8 || C0 % 8 || C1 < 0 || C1 % 8) return fail(-42, "%s: C0 and C1 must be multiples of 8 (C0 > 0, C1 >= 0)", fn);
    const int C = C0 + C1;
    if (C % 32) return fail(-42, "%s: C = C0 + C1 = %d must be a multiple of 32 (32 groups)", fn, C);
    if (C > kGnMaxC) return fail(-42, "%s: C = %d exceeds the supported maximum of %d channels", fn, C, kGnMaxC);
    if (!x0 || (C1 && !x1)) return fail(-42, "%s: null source", fn);
    if (misaligned16(x0) || misaligned16(x1)) return fail(-42, "%s: sources must be 16-byte aligned", fn);
    return 0;
}

long long ddpm_gn_scratch_bytes(int B, int C) {
    if (B < 1 || C < 1) return fail(-42, "ddpm_gn_scratch_bytes: need B >= 1 and C >= 1");
    const size_t f = gn_fwd_scratch(B), b = gn_bwd_scratch(B, C);
    return (long long)(f > b ? f : b);
}

int ddpm_groupnorm_fwd_run(const ddpm_gn_desc* d, void* stream) {
    const char* fn = "ddpm_groupnorm_fwd_run";
    if (!d) return fail(-42, "%s: null descriptor", fn);
    int rc = gn_check_src(fn, d->B, d->HW, d->C0, d->C1, d->x0, d->x1);
    if (rc) return rc;
    const int C = d->C0 + d->C1, B = d->B, r = d->route;
    if (r < 1 || r > 4) return fail(-42, "%s: route must be 1 (stats + apply), 2 (small), 3 (quad statistics) or 4 (prep)", fn);
    if (r == 2 && d->HW > 64) return fail(-42, "%s: route 2 needs HW <= 64 (got %d)", fn, d->HW);
    if (r >= 3 && C % 128) return fail(-42, "%s: routes 3 and 4 need C %% 128 == 0 (got %d)", fn, C);
    if (r >= 3 && (!d->qs0 || (d->C1 && !d->qs1))) return fail(-42, "%s: routes 3 and 4 need the quad statistics qs0 / qs1", fn);
    if (!d->gamma || !d->beta || !d->K || (r != 4 && !d->y) || (r == 1 && !d->scratch)) return fail(-42, "%s: null buffer", fn);
    if (misaligned16(d->gamma) || misaligned16(d->beta) || misaligned16(d->K) || misaligned16(d->y))
        return fail(-42, "%s: gamma, beta, K and y must be 16-byte aligned", fn);
    if (!(d->drop_p >= 0.f && d->drop_p < 1.f)) return fail(-42, "%s: drop_p must be in [0, 1)", fn);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GnApply a; memset(&a, 0, sizeof a);
    a.s.x0 = static_cast<const bf16*>(d->x0); a.s.x1 = static_cast<const bf16*>(d->x1); a.s.C0 = d->C0; a.s.C1 = d->C1;
    a.K = d->K; a.y = static_cast<bf16*>(d->y); a.HW = d->HW; a.silu = d->silu ? 1 : 0; a.drop_p = d->drop_p; a.layer = d->layer; a.mask = d->mask;
    gn_arm_dropout(a.drop_p, a.seed, (unsigned long long)d->seed);
    a.gamma = d->gamma; a.beta = d->beta; a.eps = 1e-6f; a.Kout = d->K;
    if (r == 1) {
        a.gamma = nullptr; a.beta = nullptr; a.Kout = nullptr;        // the apply pass reads the K the statistics pass finalised
        uint8_t* s = static_cast<uint8_t*>(d->scratch);
        GnFin fin; fin.gamma = d->gamma; fin.beta = d->beta; fin.K = d->K; fin.eps = 1e-6f;
        fin.ticket = reinterpret_cast<int*>(s + gn_align((size_t)B * 64 * 8));
        if ((rc = launch_gn_stats(a.s, reinterpret_cast<double*>(s), B, d->HW, fin, st))) return fail(-20, "%s: %s", fn, cudaGetErrorString((cudaError_t)rc));
        rc = launch_gn_apply(a, B, st);
    } else if (r == 2) {
        rc = launch_gn_small(a, B, st);
    } else {
        a.qs0 = d->qs0; a.qs1 = d->C1 ? d->qs1 : nullptr;
        rc = r == 3 ? launch_gn_apply(a, B, st) : launch_gn_prep(a, B, st);
    }
    return rc ? fail(-20, "%s: %s", fn, cudaGetErrorString((cudaError_t)rc)) : 0;
}

int ddpm_groupnorm_bwd_run(const ddpm_gn_bwd_desc* d, void* stream) {
    const char* fn = "ddpm_groupnorm_bwd_run";
    if (!d) return fail(-42, "%s: null descriptor", fn);
    int rc = gn_check_src(fn, d->B, d->HW, d->C0, d->C1, d->x0, d->x1);
    if (rc) return rc;
    const int C = d->C0 + d->C1, B = d->B;
    if (!d->dy || !d->K || !d->gamma || !d->dgamma || !d->dbeta || !d->dx0 || (d->C1 && !d->dx1) || !d->scratch)
        return fail(-42, "%s: null buffer", fn);
    if (misaligned16(d->dy) || misaligned16(d->K) || misaligned16(d->dx0) || misaligned16(d->dx1) || misaligned16(d->addend))
        return fail(-42, "%s: dy, K, dx0, dx1 and addend must be 16-byte aligned", fn);
    if (!(d->drop_p >= 0.f && d->drop_p < 1.f)) return fail(-42, "%s: drop_p must be in [0, 1)", fn);
    if (d->drop_p > 0.f && !d->mask) return fail(-42, "%s: drop_p > 0 needs the forward's dropout mask", fn);
    if (d->cs_per_img && d->cs_ld < C) return fail(-42, "%s: cs_ld must be >= C", fn);
    GnBwd a; memset(&a, 0, sizeof a);
    a.s.x0 = static_cast<const bf16*>(d->x0); a.s.x1 = static_cast<const bf16*>(d->x1); a.s.C0 = d->C0; a.s.C1 = d->C1;
    a.dy = static_cast<const bf16*>(d->dy); a.K = d->K; a.gamma = d->gamma;
    uint8_t* s = static_cast<uint8_t*>(d->scratch);
    const size_t cs_bytes = gn_align((size_t)B * 2 * C * 4);
    a.cs = reinterpret_cast<float*>(s); a.ticket = reinterpret_cast<int*>(s + cs_bytes);
    a.PQ = reinterpret_cast<float*>(s + cs_bytes + gn_align((size_t)B * 4));
    a.dgamma = d->dgamma; a.dbeta = d->dbeta;
    a.dx0 = static_cast<bf16*>(d->dx0); a.dx1 = d->C1 ? static_cast<bf16*>(d->dx1) : nullptr; a.acc0 = d->acc0 ? 1 : 0; a.acc1 = d->acc1 ? 1 : 0;
    a.addend = static_cast<const bf16*>(d->addend); a.B = B; a.HW = d->HW; a.silu = d->silu ? 1 : 0;
    a.drop_p = d->drop_p; a.mask = d->mask; a.dn_inplace = d->dn_inplace ? 1 : 0;
    rc = launch_gn_bwd(a, d->cs_per_img, d->cs_ld, d->cs_total, d->cs_total2, static_cast<cudaStream_t>(stream));
    return rc ? fail(-20, "%s: %s", fn, cudaGetErrorString((cudaError_t)rc)) : 0;
}

int ddpm_colsum_run(const void* dy, float* per_img, int ld, float* total, float* total2, int B, int HW, int C, int C_valid, void* stream) {
    const char* fn = "ddpm_colsum_run";
    if (!dy) return fail(-42, "%s: null dy", fn);
    if (misaligned16(dy)) return fail(-42, "%s: dy must be 16-byte aligned", fn);
    if (B < 1 || HW < 1) return fail(-42, "%s: need B >= 1 and HW >= 1", fn);
    if (C < 8 || C % 8) return fail(-42, "%s: C must be a positive multiple of 8", fn);
    if (C_valid < 1 || C_valid > C) return fail(-42, "%s: need 1 <= C_valid <= C", fn);
    if (per_img && ld < C_valid) return fail(-42, "%s: ld must be >= C_valid", fn);
    const int rc = launch_colsum(static_cast<const bf16*>(dy), per_img, ld, total, total2, B, HW, C, C_valid, static_cast<cudaStream_t>(stream));
    return rc ? fail(-20, "%s: %s", fn, cudaGetErrorString((cudaError_t)rc)) : 0;
}

// ------------------------------------------------------------------------------------------------ attention core
// scratch layout.  route 3 forward: S f32 [NB][T][T].  route 3 backward: dP f32 [NB][T][T] | dS bf16 [NB][T][T].  route 1 backward:
// dS bf16 [NB][T][T].  The dS area is used only when the caller passes no d_scores.
static size_t attn_scratch(int route, int NB, int T, int backward) {
    const size_t tt = (size_t)NB * T * T;
    if (route == ATTN_ROUTE_PRODUCTS) return gn_align(tt * 4) + (backward ? gn_align(tt * 2) : 0);
    if (route == ATTN_ROUTE_FUSED && backward) return gn_align(tt * 2);
    return 0;
}
static int attn_check(const char* fn, int route, int NB, int T, int C) {
    if (route < 1 || route > 3) return fail(-43, "%s: route must be 1 (fused), 2 (t16) or 3 (products + row softmax)", fn);
    if (NB < 1 || T < 1 || C < 1) return fail(-43, "%s: need NB >= 1, T >= 1 and C >= 1", fn);
    if (NB > 65535) return fail(-43, "%s: NB = %d exceeds 65535 (one grid z slice per image)", fn, NB);
    if (C % 8) return fail(-43, "%s: C must be a multiple of 8 (got %d)", fn, C);
    if (route == ATTN_ROUTE_FUSED && !attn_fused_eligible(T, C))
        return fail(-43, "%s: route 1 (fused) needs T = 256 and C = 256 (got T = %d, C = %d)", fn, T, C);
    if (route == ATTN_ROUTE_T16 && !attn16_eligible(T, C))
        return fail(-43, "%s: route 2 (t16) needs T = 16 and C in {128, 256, 512} (got T = %d, C = %d)", fn, T, C);
    return 0;
}
static int attn_run(const char* fn, const AttnSteps& steps, void* stream) {
    for (const AttnStep& s : steps) {
        const int rc = s.run(static_cast<cudaStream_t>(stream));
        if (rc) return fail(-20, "%s: launch '%s' failed: %s", fn, s.name.c_str(), cudaGetErrorString((cudaError_t)rc));
    }
    return 0;
}

long long ddpm_attn_scratch_bytes(int route, int NB, int T, int C, int backward) {
    const char* fn = "ddpm_attn_scratch_bytes";
    const int rc = attn_check(fn, route, NB, T, C);
    if (rc) return rc;
    if (backward != 0 && backward != 1) return fail(-43, "%s: backward must be 0 or 1 (got %d)", fn, backward);
    return (long long)attn_scratch(route, NB, T, backward);
}

int ddpm_attention_fwd_run(const ddpm_attn_desc* d, void* stream) {
    const char* fn = "ddpm_attention_fwd_run";
    if (!d) return fail(-43, "%s: null descriptor", fn);
    int rc = attn_check(fn, d->route, d->NB, d->T, d->C);
    if (rc) return rc;
    if (!d->qkv || !d->out) return fail(-43, "%s: null buffer (qkv and out are required)", fn);
    if (d->route == ATTN_ROUTE_PRODUCTS && !d->probs) return fail(-43, "%s: route 3 writes the probabilities: probs is required", fn);
    if (attn_scratch(d->route, d->NB, d->T, 0) && !d->scratch)
        return fail(-43, "%s: route %d needs a scratch area of ddpm_attn_scratch_bytes bytes", fn, d->route);
    if (misaligned16(d->qkv) || misaligned16(d->out) || misaligned16(d->probs) || misaligned16(d->scratch))
        return fail(-43, "%s: qkv, out, probs and scratch must be 16-byte aligned", fn);
    AttnSteps steps;
    rc = attn_fwd_steps(steps, d->route, static_cast<const bf16*>(d->qkv), static_cast<bf16*>(d->out), static_cast<bf16*>(d->probs),
                        static_cast<float*>(d->scratch), d->NB, d->T, d->C, false);
    return rc ? rc : attn_run(fn, steps, stream);
}

int ddpm_attention_bwd_run(const ddpm_attn_bwd_desc* d, void* stream) {
    const char* fn = "ddpm_attention_bwd_run";
    if (!d) return fail(-43, "%s: null descriptor", fn);
    int rc = attn_check(fn, d->route, d->NB, d->T, d->C);
    if (rc) return rc;
    if (!d->qkv || !d->d_out || !d->d_qkv) return fail(-43, "%s: null buffer (qkv, d_out and d_qkv are required)", fn);
    if (!d->probs) return fail(-43, "%s: the backward reads the probabilities its forward wrote: probs is required", fn);
    const size_t sb = attn_scratch(d->route, d->NB, d->T, 1);
    if (sb && !d->scratch) return fail(-43, "%s: route %d needs a scratch area of ddpm_attn_scratch_bytes bytes", fn, d->route);
    if (misaligned16(d->qkv) || misaligned16(d->d_out) || misaligned16(d->probs) || misaligned16(d->d_qkv) || misaligned16(d->d_scores) ||
        misaligned16(d->scratch))
        return fail(-43, "%s: qkv, d_out, probs, d_qkv, d_scores and scratch must be 16-byte aligned", fn);
    uint8_t* s = static_cast<uint8_t*>(d->scratch);
    float* dP = d->route == ATTN_ROUTE_PRODUCTS ? reinterpret_cast<float*>(s) : nullptr;
    bf16* dS = nullptr;
    if (d->route != ATTN_ROUTE_T16)
        dS = d->d_scores ? static_cast<bf16*>(d->d_scores)
                         : reinterpret_cast<bf16*>(s + (d->route == ATTN_ROUTE_PRODUCTS ? gn_align((size_t)d->NB * d->T * d->T * 4) : 0));
    AttnSteps steps;
    rc = attn_bwd_steps(steps, d->route, static_cast<const bf16*>(d->qkv), static_cast<const bf16*>(d->d_out), static_cast<const bf16*>(d->probs),
                        dP, dS, static_cast<bf16*>(d->d_qkv), d->NB, d->T, d->C, false);
    return rc ? rc : attn_run(fn, steps, stream);
}

// ------------------------------------------------------------------------------------------------ convolutions
// scratch layout: zero area (split-K fp32 [Ho*Wo*B][Co], or the 3x3 weight gradient's fp32 [9][Co][Cin]) | packed bf16 weights |
// combined bias fp32 [Co] | pack table (PackEntry rows: the weight packs, then the gradient unpack)
struct ConvPrep {
    int op = 0, route = 0, Ho = 0, Wo = 0, Cin = 0;
    ConvArgs a; ConvChoice ch; WgradArgs w;
    long long ldp = 0;                  // row length of the packed weights
    size_t zero_b = 0, pack_b = 0, bias_b = 0, table_b = 0;
    size_t off_pack = 0, off_bias = 0, off_table = 0, total = 0;
    int n_pack = 0; bool unpack = false, comb_bias = false;
};
static int conv_prepare(const char* fn, const ddpm_conv_desc* d, ConvPrep& p) {
    if (!d) return fail(-44, "%s: null descriptor", fn);
    if (d->op < 0 || d->op > 2) return fail(-44, "%s: op must be 0 (forward), 1 (data gradient) or 2 (weight gradient)", fn);
    if (d->route < 1 || d->route > 5) return fail(-44, "%s: route must be 1 (halo), 2 (GEMM), 3 (CUDA cores), 4 (stride 2) or 5 (fold)", fn);
    if (d->B < 1 || d->H < 1 || d->W < 1) return fail(-44, "%s: need B, H and W >= 1", fn);
    if (d->B > 65535) return fail(-44, "%s: B = %d exceeds 65535", fn, d->B);
    if (d->ksize != 1 && d->ksize != 3) return fail(-44, "%s: ksize must be 1 or 3", fn);
    if (d->stride != 1 && d->stride != 2) return fail(-44, "%s: stride must be 1 or 2", fn);
    if (d->upsample != 0 && d->upsample != 1) return fail(-44, "%s: upsample must be 0 or 1", fn);
    if ((d->identity_skip != 0 && d->identity_skip != 1) || (d->accumulate != 0 && d->accumulate != 1) || (d->dry != 0 && d->dry != 1))
        return fail(-44, "%s: identity_skip, accumulate and dry must be 0 or 1", fn);
    if (d->Cin0 < 8 || d->Cin0 % 8 || d->Cin1 < 0 || d->Cin1 % 8 || d->Co < 8 || d->Co % 8 || d->Cs0 < 0 || d->Cs0 % 8 || d->Cs1 < 0 || d->Cs1 % 8)
        return fail(-44, "%s: channel counts must be multiples of 8 (Cin0 and Co > 0)", fn);
    if (d->Cs1 && !d->Cs0) return fail(-44, "%s: a second skip source needs a first (Cs0 > 0)", fn);
    if (d->stride == 2 && (d->ksize != 3 || d->H % 2 || d->W % 2)) return fail(-44, "%s: stride 2 needs ksize 3 and an even H and W", fn);
    if ((d->stride == 2 || d->upsample) && (d->Cin0 != d->Co || d->Cin1)) return fail(-44, "%s: the resample convs need one source with Cin0 = Co", fn);
    if (d->upsample && (d->route != CONV_ROUTE_FOLD || d->op != 0 || d->ksize != 3 || d->stride != 1))
        return fail(-44, "%s: upsample = 1 is the folded route 5 (forward of a 3x3 stride-1 conv)", fn);
    if (d->route == CONV_ROUTE_FOLD && !d->upsample) return fail(-44, "%s: route 5 (fold) needs upsample = 1", fn);
    const bool skip = d->Cs0 > 0 || d->identity_skip;
    if (skip && (d->op != 0 || d->ksize != 3 || d->stride != 1 || d->upsample)) return fail(-44, "%s: a fused skip needs the forward of a 3x3 stride-1 conv", fn);
    if (d->identity_skip && (d->Cs0 != d->Co || d->Cs1 || d->w_skip || d->skip_bias)) return fail(-44, "%s: identity_skip needs Cs0 = Co, Cs1 = 0, and no w_skip or skip_bias", fn);
    if (d->skip_bias && (!d->Cs0 || d->identity_skip || !d->bias)) return fail(-44, "%s: skip_bias needs a 1x1 skip and a bias", fn);
    if (d->op == 1 && d->Cin1) return fail(-44, "%s: the data gradient writes one dx tensor: Cin1 must be 0", fn);
    if (d->op != 0 && (d->bias || d->rowvec || d->residual || d->qstats)) return fail(-44, "%s: gradients take no bias, rowvec, residual or qstats", fn);
    if (d->op == 2 && d->accumulate) return fail(-44, "%s: the weight gradient takes no accumulate flag", fn);
    if (d->rowvec && d->rowvec_ld < d->Co) return fail(-44, "%s: rowvec_ld must be >= Co", fn);
    if (!d->out || (d->op != 1 && (!d->x0 || (d->Cin1 && !d->x1))) || (d->op != 0 && !d->dy) || (d->op != 2 && !d->w) ||
        (d->Cs0 && !d->s0) || (d->Cs1 && !d->s1) || (d->Cs0 && !d->identity_skip && !d->w_skip))
        return fail(-44, "%s: null buffer", fn);
    for (const void* q : {d->x0, d->x1, d->s0, d->s1, d->dy, (const void*)d->w, (const void*)d->w_skip, (const void*)d->bias, (const void*)d->skip_bias,
                          (const void*)d->rowvec, d->residual, (const void*)d->out, (const void*)d->qstats, (const void*)d->scratch})
        if (misaligned16(q)) return fail(-44, "%s: buffers must be 16-byte aligned", fn);
    p.op = d->op; p.route = d->route; p.Cin = d->Cin0 + d->Cin1;
    p.Ho = d->upsample ? 2 * d->H : d->H / d->stride; p.Wo = d->upsample ? 2 * d->W : d->W / d->stride;
    const int taps = d->ksize * d->ksize, B = d->B;
    const bf16* x0 = static_cast<const bf16*>(d->x0); const bf16* x1 = static_cast<const bf16*>(d->x1);
    const bf16* dy = static_cast<const bf16*>(d->dy);
    int want = 0;                       // the planner's route for the shape
    if (d->op == 2) {
        WgradArgs& w = p.w;
        w.dy = dy; w.B = B; w.Ho = p.Ho; w.Wo = p.Wo; w.Co = d->Co; w.Co_valid = d->Co;
        w.in.x0 = x0; w.in.C0 = d->Cin0; w.in.x1 = d->Cin1 ? x1 : nullptr; w.in.C1 = d->Cin1; w.Hi = d->H; w.Wi = d->W;
        w.ksize = d->ksize; w.stride = d->stride; w.map = MAP_NORMAL; w.dw = static_cast<float*>(d->out);
        const bool tc = wgrad_route_tc(w);
        want = !tc ? CONV_ROUTE_SIMT : (d->stride == 2 ? CONV_ROUTE_S2 : CONV_ROUTE_GEMM);
        p.ch.route = want; p.ch.block_n = 64;
        if (tc) p.ch.splits = wgrad_splits(w, d->Cin0, &p.ch.block_n);
        if (tc && taps == 9) { p.zero_b = gn_align((size_t)9 * d->Co * p.Cin * 4); p.unpack = true; }
    } else if (d->op == 0 && d->upsample) {
        want = conv_fold_ok(d->Co, d->H, d->W) ? CONV_ROUTE_FOLD : 0;
        if (!want) return fail(-44, "%s: route 5 (fold) needs Co %% 256 == 0 and an input map the tensor-core tiles cover (got %dx%d, Co = %d)", fn, d->H, d->W, d->Co);
        p.ch.route = want; p.ch.block_n = pick_block_n(d->Co);
        p.ldp = 16LL * d->Co; p.pack_b = gn_align((size_t)d->Co * p.ldp * 2); p.n_pack = 1;
    } else if (d->op == 1 && d->stride == 2) {
        const bool tc = conv_s2_dgrad_tc(d->Co, d->H, d->W);
        want = tc ? CONV_ROUTE_S2 : CONV_ROUTE_SIMT;
        p.ch.route = want; p.ch.block_n = tc ? pick_block_n(d->Co) : 64;
        ConvArgs& a = p.a;                              // (CUDA cores: the transposed map over dY)
        a.in.x0 = dy; a.in.C0 = d->Co; a.B = B; a.Hi = p.Ho; a.Wi = p.Wo; a.ksize = 3; a.map = MAP_TRANSPOSED2;
        a.out = static_cast<bf16*>(d->out); a.Co = d->Cin0; a.Ho = d->H; a.Wo = d->W; a.accumulate = d->accumulate != 0;
        p.ldp = 9LL * d->Co; p.pack_b = gn_align((size_t)d->Cin0 * p.ldp * 2); p.n_pack = 1;
    } else {
        ConvArgs& a = p.a;
        a.B = B; a.ksize = d->ksize; a.stride = d->stride; a.map = MAP_NORMAL;
        a.out = static_cast<bf16*>(d->out); a.accumulate = d->accumulate != 0;
        if (d->op == 0) {
            a.in.x0 = x0; a.in.C0 = d->Cin0; a.in.x1 = d->Cin1 ? x1 : nullptr; a.in.C1 = d->Cin1; a.Hi = d->H; a.Wi = d->W;
            a.Co = d->Co; a.Ho = p.Ho; a.Wo = p.Wo;
            a.has_skip = skip; a.skip_identity = d->identity_skip != 0;
            a.skip.x0 = static_cast<const bf16*>(d->s0); a.skip.C0 = d->Cs0; a.skip.x1 = d->Cs1 ? static_cast<const bf16*>(d->s1) : nullptr; a.skip.C1 = d->Cs1;
            a.rowvec = d->rowvec; a.rowvec_ld = d->rowvec_ld; a.residual = static_cast<const bf16*>(d->residual);
            p.ldp = (long long)taps * p.Cin + d->Cs0 + d->Cs1; p.pack_b = gn_align((size_t)d->Co * p.ldp * 2);
            p.n_pack = 1 + (skip ? 1 : 0);
            if (d->skip_bias) { p.comb_bias = true; p.bias_b = gn_align((size_t)d->Co * 4); ++p.n_pack; }
        } else {                                        // stride-1 data gradient: a conv over dY with the transposed (3x3: flipped) weights
            a.in.x0 = dy; a.in.C0 = d->Co; a.Hi = d->H; a.Wi = d->W; a.Co = d->Cin0; a.Ho = d->H; a.Wo = d->W;
            p.ldp = (long long)taps * d->Co; p.pack_b = gn_align((size_t)d->Cin0 * p.ldp * 2); p.n_pack = 1;
        }
        p.ch = conv_choose(a, d->route != CONV_ROUTE_GEMM, true);
        want = p.ch.route;
        if (p.ch.splits > 1) p.zero_b = gn_align((size_t)B * p.Ho * p.Wo * a.Co * 4);
    }
    if (d->route != want)
        return fail(-44, "%s: route %d is not the route the planner takes for this shape (it takes route %d)", fn, d->route, want);
    if (d->qstats) {
        const bool route_ok = d->op == 0 && p.route != CONV_ROUTE_SIMT && p.ch.splits == 1;
        const int hw = d->upsample ? d->H * d->W : p.Ho * p.Wo;
        if (!route_ok || d->Co % 32 || hw % 32)
            return fail(-44, "%s: qstats needs a forward on routes 1, 2 or 4 without split-K, or route 5, with Co %% 32 == 0 and a per-image pixel count %% 32 == 0", fn);
    }
    const int n_table = p.n_pack + (p.unpack ? 1 : 0);
    p.table_b = gn_align((size_t)n_table * sizeof(PackEntry));
    p.off_pack = p.zero_b; p.off_bias = p.off_pack + p.pack_b; p.off_table = p.off_bias + p.bias_b; p.total = p.off_table + p.table_b;
    if (!d->dry && p.total && !d->scratch) return fail(-44, "%s: needs a scratch area of ddpm_conv_scratch_bytes bytes", fn);
    return 0;
}

long long ddpm_conv_scratch_bytes(const ddpm_conv_desc* d) {
    ConvPrep p;
    if (!d) return fail(-44, "ddpm_conv_scratch_bytes: null descriptor");
    ddpm_conv_desc q = *d; q.dry = 1;                  // sizes only: no scratch needed yet
    const int rc = conv_prepare("ddpm_conv_scratch_bytes", &q, p);
    return rc ? rc : (long long)p.total;
}

int ddpm_conv_run(const ddpm_conv_desc* d, void* stream) {
    const char* fn = "ddpm_conv_run";
    ConvPrep p;
    int rc = conv_prepare(fn, d, p);
    if (rc) return rc;
    uint8_t* s = static_cast<uint8_t*>(d->scratch);
    const bool dry = d->dry != 0;
    float* zero = reinterpret_cast<float*>(s);
    bf16* packed = reinterpret_cast<bf16*>(s + p.off_pack);
    float* comb = reinterpret_cast<float*>(s + p.off_bias);
    PackEntry* table = reinterpret_cast<PackEntry*>(s + p.off_table);
    // the weight packs and the gradient unpack, as the plans' repack and unpack rows
    std::vector<PackEntry> rows;
    const int taps = d->ksize * d->ksize, Co = d->Co;
    ConvSteps steps;
    if (p.op == 0 && p.route == CONV_ROUTE_FOLD) {
        rows.push_back(pack_upfold_entry(d->w, Co, packed, p.ldp));
        rc = conv_fold_steps(steps, static_cast<const bf16*>(d->x0), d->B, d->H, d->W, Co, packed, p.ldp, d->bias,
                             static_cast<bf16*>(d->out), d->qstats, dry);
    } else if (p.op == 0) {
        rows.push_back(pack_conv_entry(d->w, Co, p.Cin, taps, 0, packed, p.ldp, nullptr, 0, 0));
        if (d->identity_skip) rows.push_back(pack_identity_entry(packed, p.ldp, taps * p.Cin, Co));
        else if (d->Cs0) rows.push_back(pack_conv_entry(d->w_skip, Co, d->Cs0 + d->Cs1, 1, taps * p.Cin, packed, p.ldp, nullptr, 0, 0));
        if (p.comb_bias) rows.push_back(pack_bias_add_entry(comb, d->bias, d->skip_bias, Co));
        ConvArgs a = p.a; a.wp = packed; a.ldw = p.ldp; a.bias = p.comb_bias ? comb : d->bias; a.qstats = d->qstats;
        rc = conv_fwd_steps(steps, a, p.ch, zero, dry);
    } else if (p.op == 1) {
        // dgrad pack [Cin][taps x Co]: 3x3 stride 1 flipped taps, 1x1 plain, stride 2 the parity blocks (tensor cores) or plain
        const int dkind = d->stride == 2 ? (p.route == CONV_ROUTE_S2 ? 3 : 1) : (taps == 9 ? 2 : 1);
        rows.push_back(pack_conv_entry(d->w, Co, d->Cin0, taps, 0, nullptr, 0, packed, p.ldp, dkind));
        if (p.route == CONV_ROUTE_S2)
            rc = conv_s2_dgrad_steps(steps, static_cast<const bf16*>(d->dy), d->B, d->H, d->W, Co, packed, p.ldp, static_cast<bf16*>(d->out),
                                     d->accumulate != 0, dry);
        else { ConvArgs a = p.a; a.wp = packed; a.ldw = p.ldp; rc = conv_fwd_steps(steps, a, p.ch, zero, dry); }
    } else {
        PackEntry un;
        rc = wgrad_steps(steps, p.w, p.unpack ? zero : nullptr, &un, dry);
        if (p.unpack) rows.push_back(un);
    }
    if (rc) return rc;
    int launches = (p.n_pack ? 1 : 0) + (p.unpack ? 1 : 0);
    for (const ConvStep& st : steps) launches += st.launches;
    if (d->report) { d->report->route = p.route; d->report->launches = launches; d->report->block_n = p.ch.block_n; d->report->splits = p.ch.splits;
                     d->report->zero_bytes = (long long)p.zero_b; }
    if (dry) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaSuccess;
    if (!rows.empty() && (e = cudaMemcpyAsync(table, rows.data(), rows.size() * sizeof(PackEntry), cudaMemcpyHostToDevice, st)) != cudaSuccess)
        return fail(-20, "%s: pack table upload failed: %s", fn, cudaGetErrorString(e));
    if (p.n_pack) {
        launch_k(k_pack_table, dim3(128, p.n_pack), 256, 0, st, (const PackEntry*)table);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail(-20, "%s: weight pack failed: %s", fn, cudaGetErrorString(e));
    }
    for (const ConvStep& c : steps) {
        const int r = c.run(st);
        if (r) return fail(-20, "%s: launch '%s' failed: %s", fn, c.name.c_str(), cudaGetErrorString((cudaError_t)r));
    }
    if (p.unpack) {
        launch_k(k_pack_table, dim3(128, 1), 256, 0, st, (const PackEntry*)(table + p.n_pack));
        if ((e = cudaGetLastError()) != cudaSuccess) return fail(-20, "%s: gradient unpack failed: %s", fn, cudaGetErrorString(e));
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ precision / recall k-NN
static int knn_check(const char* fn, int n_rows, int n_cols, int D, int kk) {
    if (n_rows < 1 || n_cols < 1 || D < 1) return fail(-45, "%s: need n_rows >= 1, n_cols >= 1 and D >= 1", fn);
    if (kk < 0 || kk > KNN_MAX_K) return fail(-45, "%s: kk = nhood_size + 1 must be in 1..%d (nhood_size <= %d), got %d", fn, KNN_MAX_K, KNN_MAX_K - 1, kk);
    if (kk > n_cols) return fail(-45, "%s: kk = %d exceeds the %d columns", fn, kk, n_cols);
    if (n_rows > (1 << 30) || n_cols > (1 << 30)) return fail(-45, "%s: more than 2^30 rows or columns", fn);
    return 0;
}
static int knn_check_mat(const char* fn, const char* what, const void* x, long long ld, int D) {
    if (!x) return fail(-45, "%s: null %s", fn, what);
    if (misaligned16(x) || ld < D || ld % 8) return fail(-45, "%s: %s needs a 16-byte aligned base and a row pitch ld >= D with ld %% 8 == 0 (got ld = %lld, D = %d)", fn, what, ld, D);
    return 0;
}

long long ddpm_knn_scratch_bytes(int n_rows, int n_cols, int D, int kk) {
    const int rc = knn_check("ddpm_knn_scratch_bytes", n_rows, n_cols, D, kk);
    return rc ? rc : (long long)knn_plan(n_rows, n_cols, D, kk).total;
}

// ManifoldBuilder.compute_kth (precision_recall.py:156-164): kth_out[i] = the (kk)-th smallest distance from row i to all columns.
int ddpm_knn_kth(const void* rows, int n_rows, long long ld_rows, const void* cols, int n_cols, long long ld_cols, int D, int kk,
                 void* kth_out, void* scratch, long long bytes, void* stream) {
    const char* fn = "ddpm_knn_kth";
    int rc = knn_check(fn, n_rows, n_cols, D, kk);
    if (!rc && kk < 1) rc = fail(-45, "%s: kk must be >= 1", fn);
    if (!rc) rc = knn_check_mat(fn, "rows", rows, ld_rows, D);
    if (!rc) rc = knn_check_mat(fn, "cols", cols, ld_cols, D);
    if (rc) return rc;
    if (!kth_out) return fail(-45, "%s: null kth_out", fn);
    const size_t need = knn_plan(n_rows, n_cols, D, kk).total;
    if (!scratch || misaligned16(scratch) || bytes < (long long)need)
        return fail(-45, "%s: needs a 16-byte aligned scratch of ddpm_knn_scratch_bytes = %zu bytes (got %lld)", fn, need, bytes);
    return knn_launch(static_cast<const __half*>(rows), n_rows, ld_rows, static_cast<const __half*>(cols), n_cols, ld_cols, D, kk,
                      nullptr, kth_out, scratch, static_cast<cudaStream_t>(stream));
}

// calc_pr (precision_recall.py:177-206), one direction: covered[i] = any_j dist(probe i, support j) <= radii[j].
int ddpm_knn_cover(const void* probes, int n_probes, long long ld_p, const void* support, int n_support, long long ld_s, int D,
                   const void* radii, uint8_t* covered, void* scratch, long long bytes, void* stream) {
    const char* fn = "ddpm_knn_cover";
    int rc = knn_check(fn, n_probes, n_support, D, 0);
    if (!rc) rc = knn_check_mat(fn, "probes", probes, ld_p, D);
    if (!rc) rc = knn_check_mat(fn, "support", support, ld_s, D);
    if (rc) return rc;
    if (!radii || !covered) return fail(-45, "%s: null radii or covered", fn);
    const size_t need = knn_plan(n_probes, n_support, D, 0).total;
    if (!scratch || misaligned16(scratch) || bytes < (long long)need)
        return fail(-45, "%s: needs a 16-byte aligned scratch of ddpm_knn_scratch_bytes(.., kk = 0) = %zu bytes (got %lld)", fn, need, bytes);
    return knn_launch(static_cast<const __half*>(probes), n_probes, ld_p, static_cast<const __half*>(support), n_support, ld_s, D, 0,
                      static_cast<const __half*>(radii), covered, scratch, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ Fréchet Inception Distance
static int fid_check_d(const char* fn, int D) {
    if (D < 1 || D > FID_MAX_D) return fail(-46, "%s: D must be in 1..%d (got %d)", fn, FID_MAX_D, D);
    return 0;
}

long long ddpm_fid_stats_bytes(int D) {
    const int rc = fid_check_d("ddpm_fid_stats_bytes", D);
    return rc ? rc : (long long)fid_stats_bytes(D);
}

long long ddpm_fid_distance_scratch_bytes(int D) {
    const int rc = fid_check_d("ddpm_fid_distance_scratch_bytes", D);
    return rc ? rc : (long long)fid_dist_bytes(D);
}

// InceptionStatistics.forward (fid_score.py:116-135): the batch's features stay on the device; no np.cov, no Chan merge.
int ddpm_fid_stats_update(void* state, int D, const float* feats, long long n, long long ld, void* stream) {
    const char* fn = "ddpm_fid_stats_update";
    if (int rc = fid_check_d(fn, D)) return rc;
    if (!state || misaligned16(state)) return fail(-46, "%s: state must be a non-null, 16-byte aligned buffer", fn);
    if (n < 0 || n > INT_MAX) return fail(-46, "%s: n must be in 0..2^31-1 (got %lld)", fn, n);
    if (n == 0) return 0;
    if (!feats || (reinterpret_cast<uintptr_t>(feats) & 3)) return fail(-46, "%s: feats must be a non-null, 4-byte aligned fp32 buffer", fn);
    if (ld < D) return fail(-46, "%s: row pitch ld = %lld must be >= D = %d", fn, ld, D);
    const cudaError_t e = fid_stats_launch(state, D, feats, n, ld, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// InceptionStatistics.get_statistics (fid_score.py:137-142, ddof = 1) and the running values (ddof = 0).
int ddpm_fid_stats_finalize(const void* state, int D, long long n, int ddof, double* mean_out, double* cov_out, void* stream) {
    const char* fn = "ddpm_fid_stats_finalize";
    if (int rc = fid_check_d(fn, D)) return rc;
    if (!state || misaligned16(state) || !mean_out || !cov_out) return fail(-46, "%s: null or misaligned state / output", fn);
    if (ddof != 0 && ddof != 1) return fail(-46, "%s: ddof must be 0 or 1 (got %d)", fn, ddof);
    if (n <= ddof) return fail(-46, "%s: needs n > ddof (n = %lld, ddof = %d)", fn, n, ddof);
    const cudaError_t e = fid_finalize_launch(state, D, n, ddof, mean_out, cov_out, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// calc_fd / calculate_frechet_distance (fid_score.py:186-187, :269-323): no sqrtm of the non-symmetric product; see fid.cuh.
int ddpm_fid_distance(const double* mu1, const double* sigma1, const double* mu2, const double* sigma2, int D, double* out,
                      void* scratch, long long bytes, void* stream) {
    const char* fn = "ddpm_fid_distance";
    if (int rc = fid_check_d(fn, D)) return rc;
    if (!mu1 || !sigma1 || !mu2 || !sigma2 || !out) return fail(-46, "%s: null input or output", fn);
    if ((reinterpret_cast<uintptr_t>(mu1) | reinterpret_cast<uintptr_t>(sigma1) | reinterpret_cast<uintptr_t>(mu2) |
         reinterpret_cast<uintptr_t>(sigma2) | reinterpret_cast<uintptr_t>(out)) & 7)
        return fail(-46, "%s: inputs and output must be 8-byte aligned fp64 buffers", fn);
    const size_t need = fid_dist_bytes(D);
    if (!scratch || misaligned16(scratch) || bytes < (long long)need)
        return fail(-46, "%s: needs a 16-byte aligned scratch of ddpm_fid_distance_scratch_bytes = %zu bytes (got %lld)", fn, need, bytes);
    const cudaError_t e = fid_distance_launch(mu1, sigma1, mu2, sigma2, D, out, scratch, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ FID Inception-v3 forward
static bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

int ddpm_inception_num_params(void) { return (int)inc_params().size(); }

int ddpm_inception_param_info(int i, const char** name, int* ndim, int dims[4], long long* offset) {
    if (i < 0 || i >= (int)inc_params().size()) return fail(-47, "ddpm_inception_param_info: index %d out of 0..%d", i, (int)inc_params().size() - 1);
    const IncParam& p = inc_params()[i];
    if (name) *name = p.name.c_str();
    if (ndim) *ndim = p.ndim;
    if (dims) for (int k = 0; k < 4; ++k) dims[k] = p.dims[k];
    if (offset) *offset = p.offset;
    return 0;
}

int ddpm_inception_conv_info(int i, int info[11]) {
    if (i < 0 || i >= INC_NUM_CONVS || !info) return fail(-47, "ddpm_inception_conv_info: index %d out of 0..%d or null info", i, INC_NUM_CONVS - 1);
    static int lay[INC_NUM_CONVS][4];
    static const int steps = [] {
        for (auto& l : lay) l[3] = -1;
        IncWalk w;
        w.N = 1; w.layout = lay;
        inc_walk(w, 299, 299, 1, 3, [](int, int, int, int, int) {});
        return w.step;
    }();
    const IncConv& c = inc_convs()[i];
    const int v[11] = {c.cin, c.cout, c.kh, c.kw, c.stride, c.ph, c.pw, lay[i][0], lay[i][1], lay[i][2], steps == INC_NUM_CONVS ? lay[i][3] : -1};
    for (int k = 0; k < 11; ++k) info[k] = v[k];
    return 0;
}

long long ddpm_inception_packed_bytes(void) { return inc_packed_offsets().back() * 4; }

int ddpm_inception_pack(const float* raw, void* packed, void* stream) {
    const char* fn = "ddpm_inception_pack";
    if (!raw || misaligned(raw, 4)) return fail(-47, "%s: raw must be a non-null, 4-byte aligned fp32 buffer", fn);
    if (!packed || misaligned(packed, 256)) return fail(-47, "%s: packed must be a non-null, 256-byte aligned buffer", fn);
    const auto& convs = inc_convs();
    const auto& prm = inc_params();
    const auto& off = inc_packed_offsets();
    float* pk = static_cast<float*>(packed);
    for (size_t i = 0; i < convs.size(); ++i) {
        const float* f[INC_FIELDS];
        for (int k = 0; k < INC_FIELDS; ++k) f[k] = raw + prm[INC_FIELDS * i + k].offset;
        const cudaError_t e = inc_fold_launch(convs[i], f[0], f[1], f[2], f[3], f[4], pk + off[2 * i], pk + off[2 * i + 1],
                                              static_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
    }
    return 0;
}

static int inc_check_shape(const char* fn, int N, int H, int W, int resize, int last_block) {
    if (N < 1 || H < 1 || W < 1) return fail(-47, "%s: N, H, W must be >= 1 (got %d, %d, %d)", fn, N, H, W);
    if ((resize != 0 && resize != 1)) return fail(-47, "%s: resize must be 0 or 1 (got %d)", fn, resize);
    if (last_block < 0 || last_block > 3) return fail(-47, "%s: last_block must be in 0..3 (got %d)", fn, last_block);
    if ((long long)N * 3 * H * W > INT_MAX) return fail(-47, "%s: N * 3 * H * W exceeds 2^31 - 1", fn);
    return 0;
}

long long ddpm_inception_workspace_bytes(int N, int H, int W, int resize, int last_block) {
    const char* fn = "ddpm_inception_workspace_bytes";
    if (int rc = inc_check_shape(fn, N, H, W, resize, last_block)) return rc;
    IncWalk w;
    const char* why = nullptr;
    const size_t b = inc_workspace(N, H, W, resize, last_block, w, why);
    if (why) return fail(-47, "%s: %s (N %d, %d x %d, resize %d, last_block %d)", fn, why, N, H, W, resize, last_block);
    return (long long)b;
}

int ddpm_inception_forward(const void* packed, const float* x, int N, int H, int W, int resize, int normalize, int last_block,
                           float* const outs[4], float* pooled, void* ws, long long ws_bytes, void* stream) {
    const char* fn = "ddpm_inception_forward";
    if (int rc = inc_check_shape(fn, N, H, W, resize, last_block)) return rc;
    if (normalize != 0 && normalize != 1) return fail(-47, "%s: normalize must be 0 or 1 (got %d)", fn, normalize);
    if (!packed || misaligned(packed, 256)) return fail(-47, "%s: packed must be a non-null, 256-byte aligned buffer", fn);
    if (!x || misaligned(x, 4)) return fail(-47, "%s: x must be a non-null, 4-byte aligned fp32 buffer", fn);
    for (int b = 0; outs && b < 4; ++b)
        if (outs[b] && (b > last_block || misaligned(outs[b], 4)))
            return fail(-47, "%s: outs[%d] must be null or a 4-byte aligned buffer of a block <= last_block", fn, b);
    if (pooled && misaligned(pooled, 4)) return fail(-47, "%s: pooled must be 4-byte aligned", fn);
    IncWalk w;
    const char* why = nullptr;
    const size_t need = inc_workspace(N, H, W, resize, last_block, w, why);
    if (why) return fail(-47, "%s: %s (N %d, %d x %d, resize %d, last_block %d)", fn, why, N, H, W, resize, last_block);
    if (!ws || misaligned(ws, 256) || ws_bytes < (long long)need)
        return fail(-47, "%s: needs a 256-byte aligned workspace of ddpm_inception_workspace_bytes = %zu bytes (got %lld)", fn, need, ws_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* p = static_cast<uint8_t*>(ws);
    for (int b = 0; b < IncWalk::NBUF; ++b) { w.buf[b] = reinterpret_cast<float*>(p); p += inc_al256((size_t)w.need[b] * 4); }
    w.dry = false; w.packed = static_cast<const float*>(packed); w.st = st;
    w.err = inc_input_launch(x, N, H, W, resize, normalize, w.buf[IncWalk::X], st);
    inc_walk(w, H, W, resize, last_block, [&](int b, int buf, int h, int wd, int C) {
        if (!w.ok()) return;
        const float* src = w.buf[buf];
        const long long hw = (long long)h * wd;
        if (b == 3) {
            if (outs && outs[3]) w.err = launch_k(k_inc_gap, dim3(inc_grid((long long)N * C)), dim3(256), 0, st, src, N, (int)hw, C, outs[3], C);
            if (w.ok() && pooled) w.err = launch_k(k_inc_gap, dim3(inc_grid((long long)N * C)), dim3(256), 0, st, src, N, (int)hw, C, pooled, C);
            return;
        }
        if (outs && outs[b]) w.err = launch_k(k_inc_nchw, dim3(inc_grid(N * hw * C)), dim3(256), 0, st, src, N, (int)hw, C, outs[b]);
        if (w.ok() && pooled && b == last_block)
            w.err = launch_k(k_inc_gap, dim3(inc_grid((long long)N * C)), dim3(256), 0, st, src, N, (int)hw, C, pooled, C);
    });
    return w.err == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(w.err));
}

// the table entry a test conv stands for: any of the network's kernel shapes, with the caller's channel counts
static int inc_conv_check(const char* fn, const ddpm_inception_conv_desc* d, IncConv& c, size_t& scratch) {
    if (!d) return fail(-47, "%s: null descriptor", fn);
    if (d->N < 1 || d->H < 1 || d->W < 1 || d->Cin < 1 || d->Cout < 2 || (d->Cout & 1))
        return fail(-47, "%s: needs N, H, W, Cin >= 1 and an even Cout >= 2", fn);
    if (d->kh < 1 || d->kw < 1 || d->kh > 7 || d->kw > 7 || d->stride < 1 || d->stride > 2 || d->ph < 0 || d->pw < 0 || d->ph >= d->kh || d->pw >= d->kw)
        return fail(-47, "%s: kernel %d x %d, stride %d, padding (%d, %d) is outside 1..7, 1..2, 0..k-1", fn, d->kh, d->kw, d->stride, d->ph, d->pw);
    if (d->c_off < 0 || (d->c_off & 1) || (d->C_total & 1) || d->c_off + d->Cout > d->C_total)
        return fail(-47, "%s: channel slice [%d, %d) must be even-aligned inside an even C_total = %d", fn, d->c_off, d->c_off + d->Cout, d->C_total);
    c = IncConv{d->Cin, d->Cout, d->kh, d->kw, d->stride, d->ph, d->pw, ""};
    const int Ho = inc_conv_out(d->H, d->kh, d->stride, d->ph), Wo = inc_conv_out(d->W, d->kw, d->stride, d->pw);
    if (Ho < 1 || Wo < 1) return fail(-47, "%s: empty output", fn);
    if ((long long)d->N * d->H * d->W > INT_MAX / 4 || (long long)d->N * Ho * Wo > INT_MAX) return fail(-47, "%s: N * H * W too large", fn);
    scratch = inc_al256((size_t)inc_cout_pad(c.cout) * inc_kp(c) * 4) + inc_al256((size_t)inc_cout_pad(c.cout) * 4);
    return 0;
}

long long ddpm_inception_conv_scratch_bytes(const ddpm_inception_conv_desc* d) {
    IncConv c; size_t s = 0;
    if (int rc = inc_conv_check("ddpm_inception_conv_scratch_bytes", d, c, s)) return rc;
    return (long long)s;
}

int ddpm_inception_conv_run(const ddpm_inception_conv_desc* d, void* stream) {
    const char* fn = "ddpm_inception_conv_run";
    IncConv c; size_t s = 0;
    if (int rc = inc_conv_check(fn, d, c, s)) return rc;
    if (!d->x || misaligned(d->x, 16)) return fail(-47, "%s: x must be a non-null, 16-byte aligned buffer", fn);
    if (!d->w || !d->gamma || !d->beta || !d->mean || !d->var || !d->out) return fail(-47, "%s: null parameter or output", fn);
    if (misaligned(d->out, 8)) return fail(-47, "%s: out must be 8-byte aligned", fn);
    if (!d->scratch || misaligned(d->scratch, 256) || d->scratch_bytes < (long long)s)
        return fail(-47, "%s: needs a 256-byte aligned scratch of ddpm_inception_conv_scratch_bytes = %zu bytes (got %lld)", fn, s, d->scratch_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* wp = static_cast<float*>(d->scratch);
    float* bp = wp + inc_al256((size_t)inc_cout_pad(c.cout) * inc_kp(c) * 4) / 4;
    cudaError_t e = inc_fold_launch(c, d->w, d->gamma, d->beta, d->mean, d->var, wp, bp, st);
    if (e == cudaSuccess) e = inc_conv_launch(c, d->x, d->N, d->H, d->W, wp, bp, d->out, d->c_off, d->C_total, st);
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

int ddpm_inception_pool_run(int kind, const float* x, int N, int H, int W, int C, float* out, int c_off, int C_total, void* stream) {
    const char* fn = "ddpm_inception_pool_run";
    if (kind < 0 || kind > 2) return fail(-47, "%s: kind must be 0, 1 or 2 (got %d)", fn, kind);
    if (N < 1 || H < 1 || W < 1 || C < 1 || (long long)N * H * W * C > INT_MAX) return fail(-47, "%s: bad shape", fn);
    if (c_off < 0 || c_off + C > C_total) return fail(-47, "%s: channel slice outside C_total", fn);
    int Ho, Wo;
    inc_pool_dims(kind, H, W, Ho, Wo);
    if (Ho < 1 || Wo < 1) return fail(-47, "%s: empty output", fn);
    if (!x || !out || misaligned(x, 4) || misaligned(out, 4)) return fail(-47, "%s: null or misaligned buffer", fn);
    const cudaError_t e = inc_pool_launch(kind, x, N, H, W, C, out, c_off, C_total, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

int ddpm_inception_input_run(const float* x, int N, int H, int W, int resize, int normalize, float* out, void* stream) {
    const char* fn = "ddpm_inception_input_run";
    if (int rc = inc_check_shape(fn, N, H, W, resize, 0)) return rc;
    if (normalize != 0 && normalize != 1) return fail(-47, "%s: normalize must be 0 or 1 (got %d)", fn, normalize);
    if (!x || !out || misaligned(x, 4) || misaligned(out, 16)) return fail(-47, "%s: null or misaligned buffer", fn);
    const cudaError_t e = inc_input_launch(x, N, H, W, resize, normalize, out, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ Inception Score
long long ddpm_is_fc_packed_bytes(void) { return (long long)is_packed_bytes(); }

int ddpm_is_fc_pack(const float* fc_weight, void* packed, void* stream) {
    const char* fn = "ddpm_is_fc_pack";
    if (!fc_weight || misaligned(fc_weight, 4)) return fail(-48, "%s: fc_weight must be a non-null, 4-byte aligned fp32 buffer", fn);
    if (!packed || misaligned(packed, 256)) return fail(-48, "%s: packed must be a non-null, 256-byte aligned buffer", fn);
    const cudaError_t e = is_pack_launch(fc_weight, static_cast<float*>(packed), static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

static int is_check_n(const char* fn, int N) {
    if (N < 1) return fail(-48, "%s: N must be >= 1 (got %d)", fn, N);
    return 0;
}

long long ddpm_is_logits_workspace_bytes(int N) {
    if (int rc = is_check_n("ddpm_is_logits_workspace_bytes", N)) return rc;
    return (long long)is_logits_ws_bytes(N);
}

int ddpm_is_logits(const void* packed, const float* feats, int N, long long ld, float* logits, void* ws, long long ws_bytes, void* stream) {
    const char* fn = "ddpm_is_logits";
    if (int rc = is_check_n(fn, N)) return rc;
    if (!packed || misaligned(packed, 256)) return fail(-48, "%s: packed must be a non-null, 256-byte aligned buffer", fn);
    if (!feats || misaligned(feats, 4)) return fail(-48, "%s: feats must be a non-null, 4-byte aligned fp32 buffer", fn);
    if (ld < IS_FEAT) return fail(-48, "%s: row pitch ld = %lld must be >= %d", fn, ld, IS_FEAT);
    if (!logits || misaligned(logits, 8)) return fail(-48, "%s: logits must be a non-null, 8-byte aligned fp32 buffer", fn);
    const size_t need = is_logits_ws_bytes(N);
    if (!ws || misaligned(ws, 256) || ws_bytes < (long long)need)
        return fail(-48, "%s: needs a 256-byte aligned workspace of ddpm_is_logits_workspace_bytes = %zu bytes (got %lld)", fn, need, ws_bytes);
    const cudaError_t e = is_logits_launch(static_cast<const float*>(packed), feats, ld, N, logits, ws, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

static int is_check_score(const char* fn, int N, int C, int splits) {
    if (C < 1) return fail(-48, "%s: C must be >= 1 (got %d)", fn, C);
    if (splits < 1 || splits > N) return fail(-48, "%s: needs 1 <= splits <= N (N = %d, splits = %d)", fn, N, splits);
    if ((long long)splits * is_chunks(N, splits) * is_col_blocks(C) > INT_MAX) return fail(-48, "%s: splits * C too large", fn);
    return 0;
}

long long ddpm_is_score_scratch_bytes(int N, int C, int splits) {
    if (int rc = is_check_score("ddpm_is_score_scratch_bytes", N, C, splits)) return rc;
    return (long long)is_score_bytes(N, C, splits);
}

int ddpm_is_score(const float* logits, int N, int C, long long ld, int splits, double* out, void* scratch, long long bytes, void* stream) {
    const char* fn = "ddpm_is_score";
    if (int rc = is_check_score(fn, N, C, splits)) return rc;
    if (!logits || misaligned(logits, 4)) return fail(-48, "%s: logits must be a non-null, 4-byte aligned fp32 buffer", fn);
    if (ld < C) return fail(-48, "%s: row pitch ld = %lld must be >= C = %d", fn, ld, C);
    if (!out || misaligned(out, 8)) return fail(-48, "%s: out must be a non-null, 8-byte aligned fp64 buffer of splits + 1 values", fn);
    const size_t need = is_score_bytes(N, C, splits);
    if (!scratch || misaligned16(scratch) || bytes < (long long)need)
        return fail(-48, "%s: needs a 16-byte aligned scratch of ddpm_is_score_scratch_bytes = %zu bytes (got %lld)", fn, need, bytes);
    const cudaError_t e = is_score_launch(logits, ld, N, C, splits, out, scratch, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ Kernel Inception Distance
static int kid_check_sizes(const char* fn, int S, int m) {
    if (S < 1) return fail(-49, "%s: S (the number of subsets) must be >= 1 (got %d)", fn, S);
    if (m < 2) return fail(-49, "%s: m (the subset size) must be >= 2 (got %d)", fn, m);
    if ((long long)S * kid_blocks(m) > INT_MAX || (long long)S * 2 * m > INT_MAX) return fail(-49, "%s: S * m too large", fn);
    return 0;
}

long long ddpm_kid_scratch_bytes(int S, int m) {
    if (int rc = kid_check_sizes("ddpm_kid_scratch_bytes", S, m)) return rc;
    return (long long)kid_bytes(S, m);
}

int ddpm_kid(const float* x, long long ldx, int n1, const float* y, long long ldy, int n2, int d, const int32_t* idx_host, int S, int m,
             int degree, double gamma, double coef0, double* out, void* scratch, long long bytes, void* stream) {
    const char* fn = "ddpm_kid";
    if (int rc = kid_check_sizes(fn, S, m)) return rc;
    if (d < 1 || d > FID_MAX_D) return fail(-49, "%s: d must be in 1..%d (got %d)", fn, FID_MAX_D, d);
    if (m > n1 || m > n2) return fail(-49, "%s: needs 2 <= m <= min(n1, n2) (m = %d, n1 = %d, n2 = %d)", fn, m, n1, n2);
    if (!x || misaligned(x, 4) || !y || misaligned(y, 4)) return fail(-49, "%s: x and y must be non-null, 4-byte aligned fp32 buffers", fn);
    if (ldx < d || ldy < d) return fail(-49, "%s: row pitches ldx = %lld, ldy = %lld must be >= d = %d", fn, ldx, ldy, d);
    if (degree < 1 || degree > KID_MAX_DEGREE) return fail(-49, "%s: degree must be in 1..%d (got %d)", fn, KID_MAX_DEGREE, degree);
    if (!idx_host) return fail(-49, "%s: idx_host must be a non-null host array of S * 2 * m indices", fn);
    if (!out || misaligned(out, 8)) return fail(-49, "%s: out must be a non-null, 8-byte aligned fp64 buffer of S + 3 values", fn);
    const size_t need = kid_bytes(S, m);
    if (!scratch || misaligned16(scratch) || bytes < (long long)need)
        return fail(-49, "%s: needs a 16-byte aligned scratch of ddpm_kid_scratch_bytes = %zu bytes (got %lld)", fn, need, bytes);
    // every index in range and distinct within its half of a subset, so the kernels never see a bad row
    std::vector<int> seen((size_t)std::max(n1, n2), -1);
    for (int h = 0; h < 2 * S; ++h) {
        const int n = h & 1 ? n2 : n1;
        const int32_t* ix = idx_host + (size_t)h * m;
        for (int i = 0; i < m; ++i) {
            const int v = ix[i];
            if (v < 0 || v >= n)
                return fail(-49, "%s: subset %d: index %d of %s is out of range 0..%d", fn, h / 2, v, h & 1 ? "iy" : "ix", n - 1);
            if (seen[v] == h) return fail(-49, "%s: subset %d: index %d repeats in %s", fn, h / 2, v, h & 1 ? "iy" : "ix");
            seen[v] = h;
        }
    }
    const cudaError_t e = kid_launch(x, ldx, y, ldy, d, idx_host, S, m, degree, gamma, coef0, out, scratch, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ UNet engine
int ddpm_unet_create(const ddpm_unet_cfg* cfg, ddpm_unet** out) { return ddpm_unet_create_ex(cfg, 1, out); }
int ddpm_unet_create_ex(const ddpm_unet_cfg* cfg, int resample_with_conv, ddpm_unet** out) {
    if (!cfg || !out) return fail(-30, "null argument");
    if (resample_with_conv != 0 && resample_with_conv != 1) return fail(-30, "resample_with_conv must be 0 or 1 (got %d)", resample_with_conv);
    if (cfg->levels < 1 || cfg->levels > 8) return fail(-30, "levels must be 1..8");
    if (cfg->hid_channels <= 0 || cfg->hid_channels % 32) return fail(-30, "hid_channels must be a positive multiple of 32");
    if (cfg->num_res_blocks < 1) return fail(-30, "num_res_blocks must be >= 1");
    ddpm_unet* h = new (std::nothrow) ddpm_unet();
    if (!h) return fail(-30, "out of host memory");
    h->e.cfg = *cfg;
    h->e.resample_with_conv = resample_with_conv != 0;
    if (h->e.cfg.temb_dim <= 0) h->e.cfg.temb_dim = 4 * cfg->hid_channels;
    h->e.register_params();
    *out = h;
    return 0;
}
void ddpm_unet_destroy(ddpm_unet* h) {
    if (!h) return;
    if (h->d_samp) cudaFree(h->d_samp);
    if (h->d_bpd) cudaFree(h->d_bpd);
    if (h->e.side_stream) { cudaStreamSynchronize(h->e.side_stream);   // a queued weight re-pack still writes into the caller's workspace
        cudaStreamDestroy(h->e.side_stream); cudaEventDestroy(h->e.ev_fork); cudaEventDestroy(h->e.ev_join); }
    for (auto& c : h->e.chunks) if (c.ev) cudaEventDestroy(c.ev);
    if (h->e.ev_pack_all) { cudaEventDestroy(h->e.ev_pack_fork); cudaEventDestroy(h->e.ev_pack_fc); cudaEventDestroy(h->e.ev_pack_all); }
    delete h;
}
int ddpm_unet_num_params(const ddpm_unet* h) { return (int)h->e.params.size(); }
int ddpm_unet_param_info(const ddpm_unet* h, int i, const char** name, int* ndim, int dims[4], long long* offset) {
    if (i < 0 || i >= (int)h->e.params.size()) return fail(-30, "param index out of range");
    const ParamInfo& p = h->e.params[i];
    if (name) *name = p.name.c_str();
    if (ndim) *ndim = p.nd;
    if (dims) for (int k = 0; k < 4; ++k) dims[k] = p.dims[k];
    if (offset) *offset = p.off;
    return 0;
}
long long ddpm_unet_flat_elems(const ddpm_unet* h) { return h->e.flat_elems; }

long long ddpm_unet_graph_epoch(const ddpm_unet* h) {
    if (!h) return fail(-30, "ddpm_unet_graph_epoch: null handle");
    return h->graph_epoch;
}
long long ddpm_unet_workspace_bytes(ddpm_unet* h, int B, int H, int W, int training) {
    UnetEngine& e = h->e;
    ++h->graph_epoch;                  // the dry plan clears the op lists
    e.P = nullptr; e.G = nullptr; e.ws = nullptr; e.planned = false;
    e.zf_cursor = e.zb_cursor = 0;
    const int rc = e.plan(B, H, W, training != 0, true);
    if (rc) return rc;
    return (long long)(e.cursor + e.zf_cursor + e.zb_cursor + 8192);
}
int ddpm_unet_plan(ddpm_unet* h, int B, int H, int W, int training, float* params_flat, float* grads_flat, void* workspace, long long workspace_bytes) {
    UnetEngine& e = h->e;
    ++h->graph_epoch;
    if (!params_flat || !workspace) return fail(-30, "params / workspace pointer is null");
    if (training && !grads_flat) return fail(-30, "training plan needs a gradient buffer");
    int rc = ddpm_runtime_check(); if (rc) return rc;
    e.planned = false; h->temb_rows = false; h->image_fwd = false;
    e.P = params_flat; e.G = grads_flat; e.ws = static_cast<uint8_t*>(workspace); e.ws_bytes = (size_t)workspace_bytes;
    e.zf_cursor = e.zb_cursor = 0;
    if ((rc = e.plan(B, H, W, training != 0, true))) return rc;
    if ((long long)(e.cursor + e.zf_cursor + e.zb_cursor + 8192) > workspace_bytes)
        return fail(-32, "workspace too small: need %lld bytes, got %lld", (long long)(e.cursor + e.zf_cursor + e.zb_cursor + 8192), workspace_bytes);
    if ((rc = e.plan(B, H, W, training != 0, false))) return rc;
    if ((long long)e.cursor > workspace_bytes) return fail(-32, "workspace overflow (internal)");
    return e.build();
}
#define NEED_PLAN(h) do { if (!(h) || !(h)->e.planned) return fail(-33, "ddpm_unet_plan has not been called"); } while (0)

int ddpm_unet_repack(ddpm_unet* h, void* stream) { NEED_PLAN(h); return h->e.repack(static_cast<cudaStream_t>(stream)); }

int ddpm_unet_forward(ddpm_unet* h, const float* x, const int64_t* t, float* eps, uint64_t dropout_seed, void* stream) {
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    h->temb_rows = false; h->image_fwd = false;
    e.x_in = x; e.t_in = reinterpret_cast<const long long*>(t); e.eps_dst = eps; e.drop_seed = dropout_seed;
    return e.run_list(e.fwd_ops, static_cast<cudaStream_t>(stream));
}
int ddpm_unet_backward(ddpm_unet* h, const float* d_eps, void* stream) { return ddpm_unet_backward_ex(h, d_eps, nullptr, 1, stream); }
int ddpm_unet_backward_ex(ddpm_unet* h, const float* d_eps, float* dx, int param_grads, void* stream) {
    if (param_grads != 0 && param_grads != 1) return fail(-30, "ddpm_unet_backward_ex: param_grads must be 0 or 1 (got %d)", param_grads);
    if (!param_grads && !dx) return fail(-30, "ddpm_unet_backward_ex: nothing to compute (param_grads = 0 and dx = NULL)");
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (!e.train) return fail(-33, "plan was built without training");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    e.deps_src = d_eps; e.dx_dst = dx; e.bwd_dx = dx != nullptr; e.bwd_params = param_grads != 0;
    const int rc = e.run_list(e.bwd_ops, st);
    e.chunks_current = e.bwd_params;
    e.dx_dst = nullptr; e.bwd_dx = false; e.bwd_params = true;
    return rc;
}
int ddpm_unet_backward_launches(const ddpm_unet* h, int want_dx, int param_grads) {
    if (!h || !h->e.train) return fail(-33, "ddpm_unet_backward_launches: no training plan");
    if ((want_dx != 0 && want_dx != 1) || (param_grads != 0 && param_grads != 1)) return fail(-30, "ddpm_unet_backward_launches: flags must be 0 or 1");
    if (!want_dx && !param_grads) return fail(-30, "ddpm_unet_backward_launches: nothing to compute (want_dx = 0 and param_grads = 0)");
    return h->e.count_bwd_launches(want_dx != 0, param_grads != 0);
}
int ddpm_train_forward(ddpm_unet* h, const float* x0, const int64_t* t, const float* noise, const float* tab_a, const float* tab_s,
                       float* losses, uint64_t dropout_seed, void* stream) {
    // the loss compares eps with the noise element for element: both must have the image's channel count
    if (h && h->e.cfg.in_channels != h->e.cfg.out_channels) return fail(-30, "ddpm_train_forward: eps prediction needs out_channels == in_channels");
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    h->temb_rows = false; h->image_fwd = false;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int per_img = e.cfg.in_channels * e.H * e.W;
    const long long total = (long long)e.B * per_img;
    float* xt = e.at<float>(e.xt_off); float* eps = e.at<float>(e.eps_off);
    (void)per_img; (void)total;
    // q_sample (diffusion.py:92-97) is in_conv's load prologue: x_t is formed on the fly (and stored once, for the backward)
    e.qs_pro = QsamplePro{noise, reinterpret_cast<const long long*>(t), tab_a, tab_s, xt};
    e.x_in = x0; e.t_in = reinterpret_cast<const long long*>(t); e.eps_dst = eps; e.drop_seed = dropout_seed;
    const int rc = e.run_list(e.fwd_ops, st);
    e.qs_pro = QsamplePro{};
    e.x_in = xt;                                       // what the backward pass reads as the network input
    if (rc) return rc;
    h->train_target = noise;
    launch_k(k_mse, e.B, 256, 0, st, eps, noise, losses, e.cfg.out_channels * e.H * e.W);
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_train_backward(ddpm_unet* h, const float* gscale, void* stream) {
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (!e.train || !h->train_target) return fail(-33, "ddpm_train_forward must precede ddpm_train_backward on a training plan");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int per_img = e.cfg.out_channels * e.H * e.W;
    const long long total = (long long)e.B * per_img;
    launch_k(k_mse_grad, grid_for(total), 256, 0, st, e.at<float>(e.eps_off), h->train_target, gscale, e.at<float>(e.deps_off), per_img, total);
    DDPM_CUDA_OK(cudaGetLastError());
    e.deps_src = e.at<float>(e.deps_off);
    e.chunks_current = true;
    return e.run_list(e.bwd_ops, st);
}

// Size a step table the handle owns for n steps.  A captured graph holds the table's address: the same length keeps the allocation
// (rewritten in place by the caller), a new one reallocates it and moves the graph epoch.
static int size_table(ddpm_unet* h, void*& table, int& len, int n, size_t bytes) {
    if (len == n) return 0;
    if (table) { cudaFree(table); table = nullptr; len = 0; }
    ++h->graph_epoch;
    DDPM_CUDA_OK(cudaMalloc(&table, bytes));
    len = n;
    return 0;
}
int ddpm_sampler_setup(ddpm_unet* h, int S, const int64_t* t_model_host, const float* coef_host) {
    if (!h || S <= 0) return fail(-30, "bad sampler setup");
    const int rc = size_table(h, h->d_samp, h->S, S, (size_t)S * 8 + (size_t)S * 6 * 4);
    if (rc) return rc;
    long long* tm = static_cast<long long*>(h->d_samp);
    DDPM_CUDA_OK(cudaMemcpy(tm, t_model_host, (size_t)S * 8, cudaMemcpyHostToDevice));
    DDPM_CUDA_OK(cudaMemcpy(tm + S, coef_host, (size_t)S * 6 * 4, cudaMemcpyHostToDevice));
    return 0;
}
int ddpm_sampler_reset(ddpm_unet* h, int first_step, void* stream) {
    NEED_PLAN(h);
    if (first_step < 0 || first_step >= h->S) return fail(-30, "first_step out of range");
    launch_k(k_set_int, 1, 1, 0, static_cast<cudaStream_t>(stream), h->e.at<int>(h->e.counter_off), first_step);
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_sampler_step(ddpm_unet* h, float* x, const float* z, uint64_t seed, void* stream) {
    return ddpm_sampler_step_pred(h, x, z, seed, nullptr, stream);
}
int ddpm_sampler_step_pred(ddpm_unet* h, float* x, const float* z, uint64_t seed, float* pred_x0, void* stream) {
    // the step updates x_t in place from eps: both must have the image's channel count
    if (h && h->e.cfg.in_channels != h->e.cfg.out_channels) return fail(-30, "ddpm_sampler_step: eps prediction needs out_channels == in_channels");
    NEED_PLAN(h);
    if (!h->d_samp) return fail(-33, "ddpm_sampler_setup has not been called");
    UnetEngine& e = h->e;
    h->temb_rows = false; h->image_fwd = false;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    long long* tbuf = e.at<long long>(e.tbuf_off); float* cc = e.at<float>(e.coefcur_off); float* eps = e.at<float>(e.eps_off);
    const long long* tm = static_cast<const long long*>(h->d_samp);
    launch_k(k_sampler_prep, 1, 256, 0, st, e.at<int>(e.counter_off), tm, reinterpret_cast<const float*>(tm + h->S), 6, tbuf, cc, e.B);
    DDPM_CUDA_OK(cudaGetLastError());
    e.x_in = x; e.t_in = tbuf; e.eps_dst = eps; e.drop_seed = 0;
    static const bool no_uni = getenv("DDPM_NO_UNIFORM_T") != nullptr;
    e.uniform_t = !no_uni;                                // the whole batch is at the same timestep (diffusion.py:166)
    // the alpha/beta update of diffusion.py:107-158 rides in the epilogue of the final conv (k_out_gather): eps never reaches
    // memory and the step has no tail launch.  (Plans whose out_conv is not on the tensor-core path keep the separate tail.)
    const bool fused = e.gather_fused_tail;
    if (fused) { e.ps_epi.x = x; e.ps_epi.z = z; e.ps_epi.coef = cc; e.ps_epi.seed = (unsigned long long)seed; e.ps_epi.pred = pred_x0; }
    const int rc = e.run_list(e.fwd_ops, st);
    e.uniform_t = false;
    e.ps_epi = PsampleEpi{nullptr, nullptr, nullptr, 0, nullptr};
    if (rc) return rc;
    if (!fused) {
        const long long total = (long long)e.B * e.cfg.out_channels * e.H * e.W;
        launch_k(k_psample_tail, grid_for(total), 256, 0, st, eps, x, z, cc, (unsigned long long)seed, total, pred_x0);
        DDPM_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int ddpm_bpd_setup(ddpm_unet* h, int T, const float* coef_host) {
    if (!h || !coef_host) return fail(-30, "ddpm_bpd_setup: null argument");
    if (T <= 0 || T > (1 << 24)) return fail(-30, "ddpm_bpd_setup: T must be in 1..2^24 (the step index travels as a float)");
    const size_t bytes = (size_t)T * 8 + (size_t)T * (kBpdRow + 2) * 4;
    std::vector<uint8_t> host(bytes);
    long long* tm = reinterpret_cast<long long*>(host.data());
    float* rows = reinterpret_cast<float*>(tm + T); float* ta = rows + (size_t)T * kBpdRow; float* ts = ta + T;
    for (int i = 0; i < T; ++i) {
        tm[i] = i;
        for (int k = 0; k < kBpdRow; ++k) rows[(size_t)i * kBpdRow + k] = coef_host[(size_t)i * kBpdRow + k];
        ta[i] = coef_host[(size_t)i * kBpdRow + 0];       // the q_sample prologue indexes its tables by t
        ts[i] = coef_host[(size_t)i * kBpdRow + 1];
    }
    const int rc = size_table(h, h->d_bpd, h->bpd_T, T, bytes);
    if (rc) return rc;
    DDPM_CUDA_OK(cudaMemcpy(h->d_bpd, host.data(), bytes, cudaMemcpyHostToDevice));
    return 0;
}
int ddpm_bpd_reset(ddpm_unet* h, int first_step, void* stream) {
    NEED_PLAN(h);
    if (!h->d_bpd) return fail(-33, "ddpm_bpd_setup has not been called");
    if (first_step < 0 || first_step >= h->bpd_T) return fail(-30, "first_step out of range");
    launch_k(k_set_int, 1, 1, 0, static_cast<cudaStream_t>(stream), h->e.at<int>(h->e.counter_off), first_step);
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_bpd_step(ddpm_unet* h, const float* x0, const float* noise, int clip_denoised, float* losses, float* mses, void* stream) {
    if (!h) return fail(-30, "ddpm_bpd_step: null handle");
    if (!x0 || !noise || !losses || !mses) return fail(-30, "ddpm_bpd_step: null buffer");
    NEED_PLAN(h);
    if (!h->d_bpd) return fail(-33, "ddpm_bpd_setup has not been called");
    UnetEngine& e = h->e;
    h->temb_rows = false; h->image_fwd = false;
    const int Cin = e.cfg.in_channels, Cout = e.cfg.out_channels, HW = e.H * e.W, T = h->bpd_T;
    if (Cin != Cout) return fail(-30, "ddpm_bpd_step: eps prediction needs out_channels == in_channels");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long* tm = static_cast<const long long*>(h->d_bpd);
    const float* rows = reinterpret_cast<const float*>(tm + T); const float* ta = rows + (size_t)T * kBpdRow; const float* ts = ta + T;
    long long* tbuf = e.at<long long>(e.tbuf_off); float* cc = e.at<float>(e.coefcur_off);
    float* xt = e.at<float>(e.xt_off); float* eps = e.at<float>(e.eps_off); float* part = e.at<float>(e.bpd_part_off);
    launch_k(k_sampler_prep, 1, 256, 0, st, e.at<int>(e.counter_off), tm, rows, kBpdRow, tbuf, cc, e.B);
    DDPM_CUDA_OK(cudaGetLastError());
    // x_t = q_sample(x_0, t, noise) (diffusion.py:92-97) is formed in in_conv's loads and stored once to xt; the plain
    // forward follows (no one-row timestep path), so eps equals what ddpm_unet_forward(x_t, t) computes
    e.qs_pro = QsamplePro{noise, tbuf, ta, ts, xt};
    e.x_in = x0; e.t_in = tbuf; e.eps_dst = eps; e.drop_seed = 0;
    const BpdEpi bp{x0, xt, cc, part, clip_denoised ? 1 : 0};
    const bool fused = e.gather_fused_tail;
    if (fused) e.bpd_epi = bp;                         // eps never reaches memory
    const int rc = e.run_list(e.fwd_ops, st);
    e.qs_pro = QsamplePro{};
    e.bpd_epi = BpdEpi{};
    if (rc) return rc;
    const int nbi = (HW + 255) / 256;
    if (!fused) {
        switch (Cout) {
            case 1: launch_k(k_bpd_tail<1>, e.B * nbi, 256, 0, st, (const float*)eps, bp, HW); break;
            case 2: launch_k(k_bpd_tail<2>, e.B * nbi, 256, 0, st, (const float*)eps, bp, HW); break;
            case 3: launch_k(k_bpd_tail<3>, e.B * nbi, 256, 0, st, (const float*)eps, bp, HW); break;
            default: launch_k(k_bpd_tail<4>, e.B * nbi, 256, 0, st, (const float*)eps, bp, HW); break;
        }
        DDPM_CUDA_OK(cudaGetLastError());
    }
    launch_k(k_bpd_finalize, 1, 256, 0, st, (const float*)part, nbi, e.B, (float)(Cout * HW), (const float*)cc, T, losses, mses);
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_opt_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, float* ema_shadow, long long n,
                  const ddpm_opt_cfg* c, void* state, float* norm_out, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || !c || !state || !norm_out) return fail(-40, "ddpm_opt_step: null buffer");
    if (n <= 0 || (n & 3)) return fail(-40, "ddpm_opt_step: n must be a positive multiple of 4");
    if (c->step < 1) return fail(-40, "ddpm_opt_step: step is 1-based");
    if (c->ema_decay >= 0 && !ema_shadow) return fail(-40, "ddpm_opt_step: EMA enabled but ema_shadow is NULL");
    for (const void* q : {(const void*)params, (const void*)grads, (const void*)exp_avg, (const void*)exp_avg_sq, (const void*)ema_shadow})
        if (reinterpret_cast<uintptr_t>(q) & 15) return fail(-40, "ddpm_opt_step: buffers must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    OptScalars o;
    const double bc1 = 1.0 - pow(c->beta1, (double)c->step), bc2 = 1.0 - pow(c->beta2, (double)c->step);
    o.one_minus_b1 = (float)(1.0 - c->beta1); o.b2 = (float)c->beta2; o.one_minus_b2 = (float)(1.0 - c->beta2);
    o.step_size = (float)(c->lr / bc1); o.bc2_sqrt = (float)sqrt(bc2); o.eps = (float)c->eps;
    o.max_norm = (float)c->max_grad_norm;
    if (c->ema_decay >= 0) {
        const double nu = (double)c->ema_num_updates;
        double d = (1.0 + nu) / (10.0 + nu); if (d > c->ema_decay) d = c->ema_decay;
        o.ema_w = (float)(1.0 - d);
    } else o.ema_w = -1.f;
    static int num_sms = 0;
    if (!num_sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev); if (num_sms <= 0) num_sms = kPlanSms; }
    const long long n4 = n >> 2;
    long long want = (n4 + 255) / 256; const int cap = num_sms * 8; const int grid = (int)(want < cap ? want : cap);
    double* acc = reinterpret_cast<double*>(state); unsigned int* ticket = reinterpret_cast<unsigned int*>(acc + 1);
    launch_k(k_grad_sumsq, grid, 256, 0, st, reinterpret_cast<const float4*>(grads), n4, acc, ticket, norm_out, o.max_norm);
    DDPM_CUDA_OK(cudaGetLastError());
    launch_k(k_adam_ema, grid, 256, 0, st, reinterpret_cast<float4*>(params), reinterpret_cast<const float4*>(grads), reinterpret_cast<float4*>(exp_avg),
             reinterpret_cast<float4*>(exp_avg_sq), reinterpret_cast<float4*>(ema_shadow), n4, o, (const float*)norm_out);
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_to_uint8_nhwc(const float* x, uint8_t* out, int B, int C, int H, int W, void* stream) {
    if (!x || !out) return fail(-41, "ddpm_to_uint8_nhwc: null buffer");
    if (B <= 0 || H <= 0 || W <= 0 || C < 1 || C > 4) return fail(-41, "ddpm_to_uint8_nhwc: need B,H,W > 0 and 1 <= C <= 4");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long npix = (long long)B * H * W;
    const int grid = (int)((npix + 255) / 256 < kPlanSms * 16 ? (npix + 255) / 256 : kPlanSms * 16);
    switch (C) {
        case 1: launch_k(k_to_uint8_nhwc<1>, grid, 256, 0, st, x, out, npix, H * W); break;
        case 2: launch_k(k_to_uint8_nhwc<2>, grid, 256, 0, st, x, out, npix, H * W); break;
        case 3: launch_k(k_to_uint8_nhwc<3>, grid, 256, 0, st, x, out, npix, H * W); break;
        default: launch_k(k_to_uint8_nhwc<4>, grid, 256, 0, st, x, out, npix, H * W); break;
    }
    DDPM_CUDA_OK(cudaGetLastError());
    return 0;
}
int ddpm_unet_grad_chunks(const ddpm_unet* h, int max_n, long long* lo, long long* hi) {
    if (!h || !h->e.planned || !h->e.train) return fail(-33, "ddpm_unet_grad_chunks: no training plan");
    const int n = (int)h->e.chunks.size();
    for (int i = 0; i < n && i < max_n; ++i) { if (lo) lo[i] = h->e.chunks[i].lo; if (hi) hi[i] = h->e.chunks[i].hi; }
    return n;
}
int ddpm_unet_wait_grad_chunk(ddpm_unet* h, int i, void* stream) {
    NEED_PLAN(h);
    if (i < 0 || i >= (int)h->e.chunks.size() || !h->e.chunks[i].ev) return fail(-30, "gradient chunk index out of range");
    if (!h->e.chunks_current) return fail(-33, "the most recent backward computed no parameter gradients: it recorded no gradient chunk");
    DDPM_CUDA_OK(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), h->e.chunks[i].ev, 0));
    return 0;
}
int ddpm_unet_plan_stats(const ddpm_unet* h, int* n_fwd, int* n_bwd, int* n_tc, int* n_gen, double* ff, double* bf) {
    if (n_fwd) *n_fwd = (int)h->e.fwd_ops.size();
    if (n_bwd) *n_bwd = (int)h->e.bwd_ops.size();
    if (n_tc) *n_tc = h->e.n_tc_gemms;
    if (n_gen) *n_gen = h->e.n_generic;
    if (ff) *ff = h->e.fwd_flops;
    if (bf) *bf = h->e.bwd_flops;
    return 0;
}
int ddpm_unet_launches_per_forward(const ddpm_unet* h) { return UnetEngine::count_launches(h->e.fwd_ops); }
int ddpm_unet_launch_counts(const ddpm_unet* h, int* fwd, int* bwd, int* pack) {
    if (fwd) *fwd = UnetEngine::count_launches(h->e.fwd_ops);
    if (bwd) *bwd = h->e.count_bwd_launches(false, true);     // the default backward (no dx)
    if (pack) *pack = UnetEngine::count_launches(h->e.pack_ops);
    return 0;
}

// ------------------------------------------------------------------------------------------------ timestep-path probes
int ddpm_unet_temb_layout(const ddpm_unet* h, int max_n, int* route, int* has_uniform, int* E, int* tp_ld, int* maxc,
                          int* off, int* cout, const char** block) {
    if (!h) return fail(-30, "ddpm_unet_temb_layout: null handle");
    const UnetEngine& e = h->e;
    if (e.temb.E <= 0) return fail(-33, "ddpm_unet_temb_layout: no plan (ddpm_unet_workspace_bytes or ddpm_unet_plan first)");
    if (route) *route = e.temb.tc ? 1 : 0;
    if (has_uniform) *has_uniform = e.temb_uni_ops.empty() ? 0 : 1;
    if (E) *E = e.temb.E;
    if (tp_ld) *tp_ld = e.temb.tp_ld;
    if (maxc) *maxc = e.temb.maxc;
    const int n = (int)e.fc_table_host.size();
    for (int i = 0; i < n && i < max_n; ++i) {
        if (off) off[i] = e.fc_table_host[i].off;
        if (cout) cout[i] = e.fc_table_host[i].cout;
        if (block) block[i] = e.tp_block_host[i].c_str();
    }
    return n;
}

int ddpm_unet_temb_forward(ddpm_unet* h, const int64_t* t, int uniform, float* emb, float* e0, float* e1, float* tp, void* stream) {
    if (!h) return fail(-30, "ddpm_unet_temb_forward: null handle");
    if (!t) return fail(-30, "ddpm_unet_temb_forward: null t");
    if (uniform != 0 && uniform != 1) return fail(-30, "ddpm_unet_temb_forward: uniform must be 0 or 1 (got %d)", uniform);
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (uniform && e.temb_uni_ops.empty()) return fail(-30, "ddpm_unet_temb_forward: this plan has no one-row timestep route");
    // the forward's own zero op, then its timestep ops, or the one-row ops run_list swaps in for them under uniform_t
    std::vector<Op> ops;
    for (const Op& o : e.fwd_ops) if (o.name == "zero.fwd") ops.push_back(o);
    if (ops.size() != 1) return fail(-31, "ddpm_unet_temb_forward: internal: the plan has no 'zero.fwd' op");
    if (uniform) ops.insert(ops.end(), e.temb_uni_ops.begin(), e.temb_uni_ops.end());
    else for (const Op& o : e.fwd_ops) if (o.tag == OP_TEMB) ops.push_back(o);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    h->temb_rows = false; h->image_fwd = false;
    e.t_in = reinterpret_cast<const long long*>(t);
    int rc = e.run_list(ops, st);           // honours Op::wait_pack: the tensor-core projection waits for a pending repack
    if (rc) return rc;
    const size_t Bn = (size_t)e.B, E_ = (size_t)e.temb.E;
    const struct { float* dst; const float* src; size_t n; } cp[] = {
        {emb, e.temb.emb, Bn * e.cfg.hid_channels}, {e0, e.temb.e0, Bn * E_}, {e1, e.temb.e1, Bn * E_}, {tp, e.temb.TP, Bn * e.temb.tp_ld}};
    for (const auto& c : cp)
        if (c.dst) DDPM_CUDA_OK(cudaMemcpyAsync(c.dst, c.src, c.n * 4, cudaMemcpyDefault, st));
    h->temb_rows = !uniform;
    return 0;
}

int ddpm_unet_temb_backward(ddpm_unet* h, const float* dtp, float* d_st, float* d_s0, void* stream) {
    if (!h) return fail(-30, "ddpm_unet_temb_backward: null handle");
    if (!dtp) return fail(-30, "ddpm_unet_temb_backward: null dTP");
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (!e.train) return fail(-33, "ddpm_unet_temb_backward: plan was built without training");
    if (!h->temb_rows) return fail(-33, "ddpm_unet_temb_backward: needs a per-row ddpm_unet_temb_forward (uniform = 0) of this plan first");
    // the backward's zero op (accumulators + the flat gradient buffer), dTP in place of what the ResBlocks deposit, then the
    // timestep ops of the backward list
    std::vector<Op> zero, ops;
    for (const Op& o : e.bwd_ops) {
        if (o.name == "zero.bwd") zero.push_back(o);
        if (o.name == "temb.dtp_cast" || o.name == "temb.proj.bwd" || o.name == "temb.mlp.bwd") ops.push_back(o);
    }
    if (zero.size() != 1 || ops.size() != (e.temb.tc ? 3u : 2u)) return fail(-31, "ddpm_unet_temb_backward: internal: timestep ops not found");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    e.bwd_params = true;
    int rc = e.run_list(zero, st);
    if (rc) return rc;
    DDPM_CUDA_OK(cudaMemcpyAsync(e.temb.dTP, dtp, (size_t)e.B * e.temb.tp_ld * 4, cudaMemcpyDefault, st));
    if ((rc = e.run_list(ops, st))) return rc;
    if (d_st) DDPM_CUDA_OK(cudaMemcpyAsync(d_st, e.temb.d_st, (size_t)e.B * e.temb.E * 4, cudaMemcpyDefault, st));
    if (d_s0) DDPM_CUDA_OK(cudaMemcpyAsync(d_s0, e.temb.d_s0, (size_t)e.B * e.temb.E * 4, cudaMemcpyDefault, st));
    return 0;
}

// ------------------------------------------------------------------------------------------------ image-side convolution probes
int ddpm_unet_image_layout(const ddpm_unet* h, int* in_route, int* in_wgrad_route, int* out_route, int* dx_route, int* h0_qstats) {
    if (!h) return fail(-30, "ddpm_unet_image_layout: null handle");
    const UnetEngine& e = h->e;
    if (e.img.in_tc < 0 || e.img.out_tc < 0) return fail(-33, "ddpm_unet_image_layout: no plan (ddpm_unet_workspace_bytes or ddpm_unet_plan first)");
    if (in_route) *in_route = e.img.in_tc;
    if (in_wgrad_route) *in_wgrad_route = e.img.in_wgrad_tc;
    if (out_route) *out_route = e.img.out_tc;
    if (dx_route) *dx_route = e.img.dx_tc;
    if (h0_qstats) *h0_qstats = e.img.h0_qs ? 1 : 0;
    return 0;
}

// the ops of `L` whose names start with `prefix` (and run for this variant of the backward), in plan order
static std::vector<Op> ops_named(const std::vector<Op>& L, const std::string& prefix, bool want_dx = false) {
    std::vector<Op> r;
    for (const Op& o : L) if (o.name.compare(0, prefix.size(), prefix) == 0 && o.runs(want_dx, true)) r.push_back(o);
    return r;
}

int ddpm_unet_image_forward(ddpm_unet* h, const float* x, const int64_t* t, const float* noise, const float* tab_a, const float* tab_s,
                            const void* a, float* xt_out, void* h0_out, double* h0_qstats_out, float* eps_out, void* stream) {
    if (!h) return fail(-30, "ddpm_unet_image_forward: null handle");
    if (!x || !a || !eps_out) return fail(-30, "ddpm_unet_image_forward: x, a and eps_out are required");
    if (noise && (!t || !tab_a || !tab_s)) return fail(-30, "ddpm_unet_image_forward: noise needs t, tab_a and tab_s");
    if (xt_out && !noise) return fail(-30, "ddpm_unet_image_forward: xt_out needs noise (x_t is formed by the q_sample prologue)");
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (h0_qstats_out && !e.img.h0_qs) return fail(-30, "ddpm_unet_image_forward: this plan computes no quad statistics of h0");
    // the forward's zero op and in_conv's ops; then out_conv.2's, which wait for a pending repack as the forward's first consumer
    // of packed weights does
    std::vector<Op> in_ops, out_ops = ops_named(e.fwd_ops, "out_conv.2");
    for (const Op& o : e.fwd_ops) if (o.name == "zero.fwd") in_ops.push_back(o);
    for (const Op& o : ops_named(e.fwd_ops, "in_conv")) in_ops.push_back(o);
    if (in_ops.size() < 2 || out_ops.empty()) return fail(-31, "ddpm_unet_image_forward: internal: image ops not found");
    out_ops.front().wait_pack = 2;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    h->temb_rows = false; h->image_fwd = false;
    float* xt = e.at<float>(e.xt_off);
    if (noise) e.qs_pro = QsamplePro{noise, reinterpret_cast<const long long*>(t), tab_a, tab_s, xt};
    e.x_in = x;
    int rc = e.run_list(in_ops, st);
    e.qs_pro = QsamplePro{};
    e.x_in = noise ? xt : x;                           // what the backward reads as the network input, as after ddpm_train_forward
    if (rc) return rc;
    const size_t P = (size_t)e.B * e.H * e.W, ch = (size_t)e.cfg.hid_channels;
    DDPM_CUDA_OK(cudaMemcpyAsync(e.img.a, a, P * ch * 2, cudaMemcpyDefault, st));
    e.eps_dst = eps_out;
    if ((rc = e.run_list(out_ops, st))) return rc;
    if (xt_out) DDPM_CUDA_OK(cudaMemcpyAsync(xt_out, xt, P * e.cfg.in_channels * 4, cudaMemcpyDefault, st));
    if (h0_out) DDPM_CUDA_OK(cudaMemcpyAsync(h0_out, e.img.h0, P * ch * 2, cudaMemcpyDefault, st));
    if (h0_qstats_out) DDPM_CUDA_OK(cudaMemcpyAsync(h0_qstats_out, e.img.h0_qs, (size_t)e.B * (ch / 4) * 2 * 8, cudaMemcpyDefault, st));
    h->image_fwd = true;
    return 0;
}

int ddpm_unet_image_backward(ddpm_unet* h, const float* d_eps, const void* dh0, float* dx_out, void* d_a_out, void* stream) {
    if (!h) return fail(-30, "ddpm_unet_image_backward: null handle");
    if (!d_eps || !dh0) return fail(-30, "ddpm_unet_image_backward: d_eps and dh0 are required");
    NEED_PLAN(h);
    UnetEngine& e = h->e;
    if (!e.train) return fail(-33, "ddpm_unet_image_backward: plan was built without training");
    if (!h->image_fwd) return fail(-33, "ddpm_unet_image_backward: needs a ddpm_unet_image_forward of this plan first");
    // the backward's zero op (accumulators + the flat gradient buffer), out_conv.2's backward ops; dh0 in place of what the first
    // ResBlocks deposit, then in_conv's (with dx_out: and the input-gradient ops)
    std::vector<Op> zero, out_ops = ops_named(e.bwd_ops, "out_conv.2"), in_ops = ops_named(e.bwd_ops, "in_conv", dx_out != nullptr);
    for (const Op& o : e.bwd_ops) if (o.name == "zero.bwd") zero.push_back(o);
    if (zero.size() != 1 || out_ops.empty() || in_ops.empty() || !e.img.d_a || !e.img.dh0)
        return fail(-31, "ddpm_unet_image_backward: internal: image ops not found");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t P = (size_t)e.B * e.H * e.W, ch = (size_t)e.cfg.hid_channels;
    e.bwd_params = true; e.bwd_dx = dx_out != nullptr; e.dx_dst = dx_out; e.deps_src = d_eps;
    auto run = [&]() -> int {                           // each run_list joins the side stream (weight gradients, unpacks, bias sums)
        int rc = e.run_list(zero, st);
        if (rc || (rc = e.run_list(out_ops, st))) return rc;
        if (d_a_out) DDPM_CUDA_OK(cudaMemcpyAsync(d_a_out, e.img.d_a, P * ch * 2, cudaMemcpyDefault, st));
        DDPM_CUDA_OK(cudaMemcpyAsync(e.img.dh0, dh0, P * ch * 2, cudaMemcpyDefault, st));
        return e.run_list(in_ops, st);
    };
    const int rc = run();
    e.dx_dst = nullptr; e.bwd_dx = false;
    return rc;
}

// ------------------------------------------------------------------------------------------------ 2-D toy denoiser (toy_mlp.cuh)
static int toy_check(const char* fn, const ddpm_toy_cfg* c, long long B) {
    if (!c) return fail(-47, "%s: null config", fn);
    if (c->mid_features != 64 && c->mid_features != 128)
        return fail(-47, "%s: mid_features = %d unsupported (native: 64 or 128, the weights stay resident in shared memory)", fn, c->mid_features);
    if (c->in_features < 1 || c->in_features > 4) return fail(-47, "%s: in_features = %d unsupported (native: 1..4)", fn, c->in_features);
    if (c->num_layers < 1) return fail(-47, "%s: num_temporal_layers must be >= 1 (got %d)", fn, c->num_layers);
    if (B < 1 || B > (1LL << 24)) return fail(-47, "%s: rows must be in 1..2^24 (got %lld)", fn, B);
    return 0;
}
static int toy_check_params(const char* fn, const ddpm_toy_params* p) {
    if (!p) return fail(-47, "%s: null parameter table", fn);
    const float* const* a = &p->in_fc_weight;
    for (int i = 0; i < 15; ++i)
        if (!a[i]) return fail(-47, "%s: parameter %d is null", fn, i);
    if (misaligned16(p->fc1_weight) || misaligned16(p->fc2_weight) || misaligned16(p->enc_weight) || misaligned16(p->t_proj_weight))
        return fail(-47, "%s: the [M][M] weights must be 16-byte aligned", fn);
    return 0;
}
static int toy_check_ws(const char* fn, const ddpm_toy_cfg* c, long long rows, int training, const void* ws, long long bytes) {
    const size_t need = toy_ws_layout(c->mid_features, c->in_features, c->num_layers, rows, training).total;
    if (!ws || (reinterpret_cast<uintptr_t>(ws) & 255) || bytes < (long long)need)
        return fail(-47, "%s: needs a 256-byte aligned workspace of ddpm_toy_workspace_bytes = %zu bytes (got %lld)", fn, need, bytes);
    return 0;
}
static ToyArgs toy_args(const ddpm_toy_cfg* c, const ddpm_toy_params* p, long long B, void* ws, int training) {
    ToyArgs a; memset(&a, 0, sizeof a);
    a.w = *p; a.M = c->mid_features; a.D = c->in_features; a.L = c->num_layers; a.B = (int)B;
    const ToyWs l = toy_ws_layout(a.M, a.D, a.L, B, training);
    uint8_t* b = static_cast<uint8_t*>(ws);
    a.E = reinterpret_cast<float*>(b + l.E);
    if (training) {
        a.h_sv = reinterpret_cast<float*>(b + l.h); a.u_sv = reinterpret_cast<float*>(b + l.u);
        a.x_sv = reinterpret_cast<float*>(b + l.x); a.out_sv = reinterpret_cast<float*>(b + l.out);
        a.dE = reinterpret_cast<float*>(b + l.dE); a.part = reinterpret_cast<float*>(b + l.part);
    }
    return a;
}
static int toy_done(const char* fn, cudaError_t e) { return e == cudaSuccess ? 0 : fail(-20, "%s: launch failed: %s", fn, cudaGetErrorString(e)); }

long long ddpm_toy_num_params(const ddpm_toy_cfg* cfg) {
    if (int rc = toy_check("ddpm_toy_num_params", cfg, 1)) return rc;
    return ToyLayout(cfg->mid_features, cfg->in_features, cfg->num_layers).P;
}

long long ddpm_toy_workspace_bytes(const ddpm_toy_cfg* cfg, long long rows, int training) {
    if (int rc = toy_check("ddpm_toy_workspace_bytes", cfg, rows)) return rc;
    return (long long)toy_ws_layout(cfg->mid_features, cfg->in_features, cfg->num_layers, rows, training ? 1 : 0).total;
}

int ddpm_toy_forward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const float* x, const long long* t, long long B, float* out,
                     int training, void* ws, long long ws_bytes, void* stream) {
    const char* fn = "ddpm_toy_forward";
    if (int rc = toy_check(fn, cfg, B)) return rc;
    if (int rc = toy_check_params(fn, p)) return rc;
    if (!x || !t || !out) return fail(-47, "%s: null x, t or out", fn);
    if (int rc = toy_check_ws(fn, cfg, B, training ? 1 : 0, ws, ws_bytes)) return rc;
    ToyArgs a = toy_args(cfg, p, B, ws, training ? 1 : 0);
    a.x = x; a.t = t; a.out = out;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return toy_done(fn, a.M == 64 ? toy_forward_launch<64>(a, st) : toy_forward_launch<128>(a, st));
}

int ddpm_toy_train_forward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const float* x0, const long long* t, const float* noise,
                           const float* sqrt_ab, const float* sqrt_1mab, long long B, float* losses, void* ws, long long ws_bytes,
                           void* stream) {
    const char* fn = "ddpm_toy_train_forward";
    if (int rc = toy_check(fn, cfg, B)) return rc;
    if (int rc = toy_check_params(fn, p)) return rc;
    if (!x0 || !t || !noise || !sqrt_ab || !sqrt_1mab || !losses) return fail(-47, "%s: null input or output", fn);
    if (int rc = toy_check_ws(fn, cfg, B, 1, ws, ws_bytes)) return rc;
    ToyArgs a = toy_args(cfg, p, B, ws, 1);
    a.x0 = x0; a.t = t; a.noise = noise; a.sa = sqrt_ab; a.s1a = sqrt_1mab; a.loss = losses;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return toy_done(fn, a.M == 64 ? toy_forward_launch<64>(a, st) : toy_forward_launch<128>(a, st));
}

static int toy_backward_common(const char* fn, const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const long long* t, long long B,
                               const float* d_out, const float* noise, const float* g, float* dx, float* grad, void* ws,
                               long long ws_bytes, void* stream) {
    if (int rc = toy_check(fn, cfg, B)) return rc;
    if (int rc = toy_check_params(fn, p)) return rc;
    if (!t || !grad || (!d_out && !(noise && g))) return fail(-47, "%s: null t, seed gradient or grad", fn);
    if (int rc = toy_check_ws(fn, cfg, B, 1, ws, ws_bytes)) return rc;
    ToyArgs a = toy_args(cfg, p, B, ws, 1);
    a.t = t; a.d_out = d_out; a.noise = noise; a.g = g; a.dx = dx;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return toy_done(fn, a.M == 64 ? toy_backward_launch<64>(a, grad, st) : toy_backward_launch<128>(a, grad, st));
}

int ddpm_toy_backward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const long long* t, const float* d_out, long long B,
                      float* dx, float* grad, void* ws, long long ws_bytes, void* stream) {
    if (!d_out) return fail(-47, "ddpm_toy_backward: null d_out");
    return toy_backward_common("ddpm_toy_backward", cfg, p, t, B, d_out, nullptr, nullptr, dx, grad, ws, ws_bytes, stream);
}

int ddpm_toy_train_backward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const long long* t, const float* noise, const float* g,
                            long long B, float* grad, void* ws, long long ws_bytes, void* stream) {
    if (!noise || !g) return fail(-47, "ddpm_toy_train_backward: null noise or g");
    return toy_backward_common("ddpm_toy_train_backward", cfg, p, t, B, nullptr, noise, g, nullptr, grad, ws, ws_bytes, stream);
}

int ddpm_toy_sample(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, float* x, long long B, int S, const float* coef,
                    const float* z, void* ws, long long ws_bytes, void* stream) {
    const char* fn = "ddpm_toy_sample";
    if (int rc = toy_check(fn, cfg, B)) return rc;
    if (int rc = toy_check_params(fn, p)) return rc;
    if (S < 1 || S > 100000) return fail(-47, "%s: S must be in 1..100000 (got %d)", fn, S);
    if (!x || !coef || !z) return fail(-47, "%s: null x, coef or z", fn);
    if (int rc = toy_check_ws(fn, cfg, S, 0, ws, ws_bytes)) return rc;
    ToyArgs a = toy_args(cfg, p, B, ws, 0);
    a.x = x; a.coef = coef; a.z = z; a.S = S;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return toy_done(fn, a.M == 64 ? toy_sample_launch<64>(a, st) : toy_sample_launch<128>(a, st));
}

}  // extern "C"
