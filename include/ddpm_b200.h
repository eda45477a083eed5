/* ddpm_b200 — C ABI of the H100-native DDPM engine (libddpm_b200.so).
 *
 * The reference (tqch/ddpm-torch @ b60eb8d) is pure Python on PyTorch and has NO FFI / plugin interface;
 * its seam for this path is the Python callable protocol  denoise_fn(x_t f32[B,C,H,W], t i64[B]) -> f32[B,C,H,W]
 * (ddpm_torch/diffusion.py:109,238; ddim.py:101) plus the GaussianDiffusion / DDIM methods that call it.
 * This header is what a ctypes binding on the reference side binds instead (see INTEGRATION.md); every entry
 * point cites the reference code it replaces.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise; the caller
 *    (PyTorch's caching allocator on the Python side) owns every buffer; the library allocates nothing per call,
 *    never synchronises, and is CUDA-graph capturable; `stream` is a cudaStream_t passed as void*.
 *  - every function returns 0 on success, <0 on error; ddpm_last_error() returns the message (thread local).
 *    No exceptions or aborts cross the ABI (the reference raises Python exceptions: diffusion.py:42-43,119,133).
 *  - activations inside the engine are NHWC bf16; the 3-channel network input/output stay NCHW fp32 exactly
 *    as the reference hands them over (unet.py:205,232).
 */
#ifndef DDPM_B200_H
#define DDPM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* ddpm_last_error(void);
/* 0 when the library was built for sm_90a and a CUDA driver + sm_90 device are present. */
int ddpm_runtime_check(void);
/* Device-side error flag set by a bounded wait that timed out inside a kernel (0 = none). Synchronises. */
int ddpm_device_error_flag(void);

/* Optional GroupNorm fusion of a conv / GEMM epilogue (nn.GroupNorm(32, C, eps=1e-6) of unet.py:18-20; csrc/gn_epilogue.cuh).
 *  qstats   the producer adds per (image, 4-channel quad) {sum, sum of squares} of its OUTPUT to qstats[NB][N/4][2]
 *           (fp64 atomics, caller zeroes it) - the statistics pass of the consuming GroupNorm disappears.  NULL = off. */
typedef struct ddpm_gn_epi {
    double* qstats;
} ddpm_gn_epi;

/* ------------------------------------------------------------------------------------------------
 * Low-level operator: one wgmma implicit-GEMM launch (used by the parity tests of the engine itself).
 * mode 0 (KK)   A K-major NHWC pixel tiles (+3x3 taps, up to 3 channel segments), B K-major matrix stack
 * mode 1 (MNMN) A,B MN-major, K over pixels (conv wgrad / P^T.dO); split-K with fp32 atomics
 * mode 2 (KMN)  A K-major, B MN-major (P.V)
 * replaces: F.conv2d (modules.py:121-123), F.linear (modules.py:59), torch.einsum x2 (unet.py:46-51) and their
 * autograd backward formulas.
 */
typedef struct ddpm_gemm_desc {
    int mode, block_n;                 /* block_n 0 = auto (64/128/256) */
    int M, N;                          /* output rows / cols per z slice */
    int W, H, NB;                      /* geometry of the NHWC tensors behind the 4-D maps (plain matrix: W=rows,H=1) */
    const void* a_ptr[3]; int a_C[3]; long long a_ld[3];   /* up to 3 A tensors: channels extent, pixel stride (elements) */
    int nseg; int seg_map[3], seg_taps[3], seg_kchunks[3], seg_cbase[3];
    const void* b_ptr; int b_K, b_rows, b_batch; long long b_ld, b_bs;  /* KK: [b_batch][b_rows][b_K]; MN modes: b_K = channel extent, b_ld = pixel stride */
    int b_k_base, a_z_n, b_z;
    int taps, splits, kblocks, a_c_base, b_c_base, grid_z;
    void* out; int ldo; long long out_z_stride, out_tap_stride; int flags;   /* flags: 1 = fp32 out, 2 = atomic add (fp32) */
    const float* bias; const float* rowvec; int rowvec_ld, rows_per_vec;
    const void* residual; int ldr; float alpha;
    /* stride-2 support: a_estride/b_estride = 2 builds the A (KK) / B (MNMN) map over a (W*2, H*2) tensor sampled with
     * elementStrides 2; seg_cmul multiplies the tile origin; seg_dx/seg_dy override the default 3x3 offsets when seg_custom != 0;
     * o_mul/o_py/o_px scatter output rows to pixel (y*o_mul+o_py, x*o_mul+o_px) of an (W*o_mul, H*o_mul) grid. */
    int a_estride, b_estride, b_pad;
    int seg_custom[3], seg_cmul[3]; signed char seg_dx[3][9], seg_dy[3][9];
    int o_mul, o_py, o_px;
    int kk_splits;                     /* mode 0: split the K loop over grid_z = kk_splits CTAs per tile (fp32 atomic output) */
    ddpm_gn_epi gn;                    /* mode 0 only, rows = NHWC pixels with H*W % 32 == 0 */
    int cta_pair;                      /* accepted for ABI compatibility and ignored: sm_90 has no CTA-pair MMA, every GEMM runs
                                        * on the single-CTA wgmma kernel */
} ddpm_gemm_desc;
int ddpm_gemm_run(const ddpm_gemm_desc* d, void* stream);

/* Low-level operator: 3x3 stride-1 convolution (+ optional fused 1x1 segments) with a haloed shared-memory input tile
 * (csrc/conv_halo.cuh) — the kernel behind ResidualBlock.conv1 / conv2(+skip) (unet.py:76,79,80) at resolutions >= 16x16.
 * a_ptr/a_C/a_ld: up to 3 NHWC bf16 inputs; segment s reads map seg_map[s] with seg_taps[s] in {9 (3x3, pad 1), 1 (1x1)},
 * seg_kchunks[s] chunks of 64 channels starting at channel seg_cbase[s]; w: packed bf16 [Cout][ldw], K order = segments,
 * then tap, then channel; out: NHWC bf16 [NB,H,W,Cout] = conv + bias + rowvec[image] + residual. */
typedef struct ddpm_halo_desc {
    int NB, H, W, Cout;
    const void* a_ptr[3]; int a_C[3]; long long a_ld[3];
    int nseg; int seg_map[3], seg_taps[3], seg_kchunks[3], seg_cbase[3];
    const void* w; long long ldw; int Ktot;
    void* out; const float* bias; const float* rowvec; int rowvec_ld; const void* residual;
    int base_offset_mode;              /* 0 = descriptor base_offset field left 0 (correct); 1 = (addr>>7)&7 (probe) */
    int force_sub;                     /* 0 = auto (one 16x8 sub-tile per CTA); 2 = two sub-tiles (W % 16 == 0, at most 128 output channels
                                        * per CTA); 1 and 3 = one sub-tile */
    ddpm_gn_epi gn;
    /* force_sub = 3 / CTA-pair kernel only: the 3x3 segment's input (map 0) is the RAW input of a GroupNorm(+SiLU); the kernel
     * applies y = act(sc*x + sh) to every landed tile in shared memory (unet.py:83-84: conv(act(norm(x)))), xf_K [NB][4][C] holding
     * {sc, sh, ...} per (image, channel).  NULL = off. */
    const float* xf_K; int xf_silu;
} ddpm_halo_desc;
int ddpm_conv_halo_run(const ddpm_halo_desc* d, void* stream);

/* Low-level operator: the attention core of AttentionBlock.forward (unet.py:43-51) as ONE kernel (csrc/attn_fused.cuh):
 * out[b] = softmax(Q K^T / sqrt(C)) V with q, k, v = the three C-channel thirds of qkv bf16 [NB][T][3C] (chunk order of unet.py:57),
 * out bf16 [NB][T][C].  S and O stay in tensor memory, P in shared memory.  Supported: T = 256 tokens (the 16x16 level), C = 256.
 * probs (optional, NULL = off): bf16 [NB][T][T], receives the softmax probabilities that the backward pass of a training plan
 * consumes (written from the shared-memory tile while P.V runs). */
int ddpm_attn_fused_run(const void* qkv, void* out, void* probs, int NB, int T, int C, void* stream);
/* Query-side half of the attention backward (autograd of unet.py:43-51) as ONE kernel: with P = probs saved by the forward,
 * dP = d_out V^T,  dS = P o (dP - rowsum(P o dP)) / sqrt(C)  -> d_scores bf16 [NB][T][T],  dQ = dS K -> the q third of
 * d_qkv bf16 [NB][T][3C].  dK = dS^T Q and dV = P^T d_out are plain GEMMs over d_scores / probs (ddpm_gemm_run).  T = 256, C = 256. */
int ddpm_attn_fused_bwd_run(const void* qkv, const void* d_out, const void* probs, void* d_scores, void* d_qkv, int NB, int T, int C, void* stream);

/* Low-level operators: the attention core softmax(Q K^T / sqrt(C)) V of AttentionBlock (unet.py:43-51) and its backward, on any
 * route the UNet engine's plans take, with the launch sequence those plans use (used by the parity tests of the engine itself).
 * Routes (the engine picks one per attention block from the shape):
 *  1  fused: attn_kernel<false>; backward attn_kernel<true> (dP, dS, dQ) + the dV and dK products.  T = 256, C = 256
 *  2  t16: k_attn16_fwd / k_attn16_bwd, one CTA per image.  T = 16, C in {128, 256, 512}
 *  3  products + row softmax: Q.K^T (fp32 S) -> k_softmax_rows -> P.V; backward dP (fp32), dV, k_softmax_bwd (dS), dQ, dK.  The
 *     products run on the tensor cores when T is a power of two, T % 128 == 0 and C % 64 == 0, on CUDA cores otherwise.  Any T.
 * qkv bf16 [NB][T][3C] (q | k | v, the chunk order of unet.py:57), out / d_out bf16 [NB][T][C], probs bf16 [NB][T][T] (forward:
 * optional on routes 1 and 2, required and always written on route 3; backward: the probabilities a forward wrote, required),
 * d_qkv bf16 [NB][T][3C] (all three thirds written), d_scores bf16 [NB][T][T] (optional; receives dS on routes 1 and 3, route 2
 * does not form it in memory).  scratch: caller-owned device area of ddpm_attn_scratch_bytes(route, NB, T, C, backward) bytes (0
 * when the route needs none: route 3's fp32 S / dP, and dS when d_scores is NULL).  C is a multiple of 8, 1 <= NB <= 65535,
 * buffers are 16-byte aligned.  Arguments are checked before any device work. */
typedef struct ddpm_attn_desc {
    int route, NB, T, C;
    const void* qkv; void* out; void* probs;
    void* scratch;
} ddpm_attn_desc;
typedef struct ddpm_attn_bwd_desc {
    int route, NB, T, C;
    const void* qkv; const void* d_out; const void* probs;
    void* d_qkv; void* d_scores;
    void* scratch;
} ddpm_attn_bwd_desc;
int ddpm_attention_fwd_run(const ddpm_attn_desc* d, void* stream);
int ddpm_attention_bwd_run(const ddpm_attn_bwd_desc* d, void* stream);
long long ddpm_attn_scratch_bytes(int route, int NB, int T, int C, int backward);

/* Low-level operator: one convolution of the UNet (unet.py:63-89,163-170,199-202: conv1, conv2 + skip, project_in / _out, the
 * resample convs), its data gradient or its weight gradient, on an explicit route, with the launch steps, descriptors and packed
 * weight layouts the UNet engine's plans use (used by the parity tests of the engine itself).
 *  op 0  forward:         out bf16 NHWC [B][Ho][Wo][Co] = conv(x) [+ 1x1 skip(s)] + bias (+ skip_bias) + rowvec[b] + residual
 *                         (accumulate != 0: out += instead of the residual)
 *  op 1  data gradient:   out = dx bf16 [B][H][W][Cin0] (=, or += with accumulate) from dy bf16 [B][Ho][Wo][Co] and the same weights
 *  op 2  weight gradient: out = dW fp32 OIHW [Co][Cin0 + Cin1][k][k] from dy and the conv input x0 | x1.  The tensor-core 1x1 and
 *                         the CUDA-core routes ADD into out (the engine's flat gradient buffer is zeroed per backward); the
 *                         tensor-core 3x3 routes write it.
 * Geometry: B, H, W of the conv input; ksize 1 or 3; stride 1 (pad ksize/2) or 2 (3x3, SamePad2d: bottom / right only, H and W
 * even, Cin0 = Co); upsample = 1 (route 5 only): nearest-2x upsample, then the 3x3 conv on the 2H x 2W grid, Cin0 = Co.
 * Output map Ho x Wo = H x W, H/2 x W/2 (stride 2) or 2H x 2W (upsample).
 * Inputs: x0 | x1 the channel concat [B][H][W][Cin0 | Cin1] (Cin1 = 0: one source; op 1 takes none); s0 | s1 [B][H][W][Cs0 | Cs1]
 * the fused 1x1 skip's concat (forward of a 3x3 stride-1 conv only), or identity_skip = 1: s0 with Cs0 = Co enters with identity
 * weights (the ResidualBlock's residual as extra K chunks).  All channel counts are multiples of 8.
 * Weights: fp32 OIHW masters w [Co][Cin0 + Cin1][k][k] and w_skip [Co][Cs0 + Cs1], packed to bf16 by the engine's pack rows
 * (k_pack_table) inside the call; bias / skip_bias [Co] (skip_bias with a 1x1 skip: added to bias by PK_BIAS_ADD); rowvec
 * [B][rowvec_ld]; residual bf16 like out.  qstats (optional) [B][Co/4][2] fp64 {sum, sum of squares} per image and channel quad of
 * the output, added to (the caller zeroes it): forward on routes 1, 2 and 4 without split-K, and route 5, with Co % 32 == 0 and
 * a pixel count per image (route 5: of the low-resolution input) that is a multiple of 32.
 * Routes, refused unless the engine's planner takes that route for the shape (route 2 as it does with the haloed kernel off):
 *  1 halo: conv_halo.cuh (3x3 stride 1, H % 16 == 0, W % 8 == 0, H >= 16)
 *  2 GEMM on the tensor cores, split over K (+ k_splitk_finalize) exactly when the planner splits; weight gradients GEMM_MNMN
 *  3 CUDA cores: k_conv_generic (+ one launch for a skip; MAP_TRANSPOSED2 for the stride-2 data gradient), k_wgrad_generic
 *  4 stride 2 on the tensor cores: the forward, the data gradient as four output-parity GEMMs, the weight gradient
 *  5 nearest-2x upsample folded into the 3x3 conv: four output-parity GEMMs over merged weights (forward only)
 * scratch: caller-owned device area of ddpm_conv_scratch_bytes(d) bytes whose first zero_bytes (see the report) must be zero on entry
 * and are zero again on return; the rest holds the packed weights and pack table.  Buffers are 16-byte aligned.
 * report (optional): what the call launches (route, kernel launches, block_n of the output tiles, split count over K of the
 * tensor-core GEMM routes).  dry = 1 fills the report and does no device work.  Every argument error is refused before any device
 * work. */
typedef struct ddpm_conv_report {
    int route, launches, block_n, splits;
    long long zero_bytes;
} ddpm_conv_report;
typedef struct ddpm_conv_desc {
    int op, route;
    int B, H, W, ksize, stride, upsample;
    int Cin0, Cin1, Co, Cs0, Cs1, identity_skip;
    const void* x0; const void* x1; const void* s0; const void* s1; const void* dy;
    const float* w; const float* w_skip;
    const float* bias; const float* skip_bias; const float* rowvec; int rowvec_ld;
    const void* residual; int accumulate;
    void* out; double* qstats;
    void* scratch;
    int dry;
    ddpm_conv_report* report;
} ddpm_conv_desc;
int ddpm_conv_run(const ddpm_conv_desc* d, void* stream);
long long ddpm_conv_scratch_bytes(const ddpm_conv_desc* d);

/* ------------------------------------------------------------------------------------------------
 * k-NN half of the improved precision/recall metric (ddpm_torch/metrics/precision_recall.py): one fp16 wgmma GEMM per pass with a
 * selection epilogue (knn.cuh), in place of the reference's fp16 cdist blocks copied to the host.  Feature matrices are fp16
 * [n][ld] (device), 16-byte aligned, ld >= D and ld % 8 == 0 (elements past D in a row are ignored).  Any D >= 1.
 *   na[i] = sum_d a[i,d]^2 (fp32);  d2[i,j] = max(0, na[i] + nb[j] - 2 <a_i, b_j>) (fp16 wgmma, fp32 accumulation)
 * ddpm_knn_kth   (compute_kth, :156-164): kth_out fp16 [n_rows] = fp16_rn(sqrt_rn(kk-th smallest d2[i, .])), all columns
 *                including row i itself when rows == cols; kk = nhood_size + 1 in 1..16 and kk <= n_cols.
 * ddpm_knn_cover (calc_pr, :177-206, one direction): covered u8 [n_probes] = 1 iff some support j has
 *                fp16_rn(sqrt_rn(d2[i,j])) <= radii[j] (fp16 [n_support]), else 0.
 * scratch: caller-owned, 16-byte aligned, ddpm_knn_scratch_bytes(n_rows, n_cols, D, kk) bytes (kk = 0 for ddpm_knn_cover); no
 * initialisation needed.  No allocation, no synchronisation, graph-capturable; results are bit-identical from call to call.  Every
 * argument error is refused before any device work. */
long long ddpm_knn_scratch_bytes(int n_rows, int n_cols, int D, int kk);
int ddpm_knn_kth(const void* rows, int n_rows, long long ld_rows, const void* cols, int n_cols, long long ld_cols, int D, int kk,
                 void* kth_out, void* scratch, long long bytes, void* stream);
int ddpm_knn_cover(const void* probes, int n_probes, long long ld_p, const void* support, int n_support, long long ld_s, int D,
                   const void* radii, uint8_t* covered, void* scratch, long long bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fréchet Inception Distance (ddpm_torch/metrics/fid_score.py), fp64 throughout, on the fp64 tensor cores (DMMA) where it is a
 * contraction (fid.cuh).  D in 1..4096.  No allocation, no synchronisation; results are bit-identical from call to call, and every
 * argument error is refused before any device work.
 * ddpm_fid_stats_update   (InceptionStatistics.forward, :116-135): folds n rows of fp32 features feats[n][ld] (device, 4-byte
 *                         aligned, ld >= D) into the state: state bytes = ddpm_fid_stats_bytes(D), 16-byte aligned, zero-filled by the
 *                         caller before the first update (and to reset).  The row count stays with the caller; n = 0 is a no-op.
 * ddpm_fid_stats_finalize (:137-142): mean f64[D] and cov f64[D][D] (full, symmetric) of the n rows folded in so far, cov divided by
 *                         n - ddof (ddof 1: get_statistics; ddof 0: the population running values).  Needs n > ddof.
 * ddpm_fid_distance       (calc_fd / calculate_frechet_distance, :186-187, :269-323): mu f64[D], sigma f64[D][D] (device);
 *                         out f64[8] (device) <- {fd, status, sweeps(sigma1), sweeps(M), lam_min/lam_max(sigma1),
 *                         nu_min/nu_max(M), tr sqrt(sigma1 sigma2), 0} with M = L^T sigma2 L, sigma1 = L L^T.  status: 0 ok,
 *                         1 non-finite input, 2 sigma1 not PSD (lam_min < -1e-6 lam_max), 3 M not PSD (sigma2 not PSD),
 *                         4 / 5 eigen-solve of sigma1 / M did not converge within 60 sweeps; fd is NaN unless status is 0.
 *                         scratch: ddpm_fid_distance_scratch_bytes(D) bytes, 16-byte aligned, no initialisation needed. */
long long ddpm_fid_stats_bytes(int D);
int ddpm_fid_stats_update(void* state, int D, const float* feats, long long n, long long ld, void* stream);
int ddpm_fid_stats_finalize(const void* state, int D, long long n, int ddof, double* mean_out, double* cov_out, void* stream);
long long ddpm_fid_distance_scratch_bytes(int D);
int ddpm_fid_distance(const double* mu1, const double* sigma1, const double* mu2, const double* sigma2, int D, double* out,
                      void* scratch, long long bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FID Inception-v3 forward (ddpm_torch/metrics/inception.py; inception.cuh): the 94 BasicConv2d layers (conv, eval BatchNorm
 * eps = 1e-3, ReLU) as TF32 implicit GEMMs on the tensor cores, the pools and the global average as SIMT kernels, NHWC fp32 inside.
 * Stateless: every buffer is the caller's, nothing is allocated, nothing synchronises, every call can be captured in a graph, and
 * every argument is checked before the first launch.  An image's outputs are bit-identical whatever batch it arrives in.
 * ddpm_inception_num_params / _param_info: the raw parameters in torchvision Inception3's state_dict key order (num_batches_tracked
 *                         and fc.* left out): 5 per conv (conv.weight [Cout][Cin][kh][kw], bn.weight, bn.bias, bn.running_mean,
 *                         bn.running_var [Cout]) at fp32 element `offset` of one flat raw buffer.  dims past ndim are 0.
 * ddpm_inception_conv_info conv i (state_dict order) as the forward runs it: {Cin, Cout, kh, kw, stride, ph, pw, c_off, C_total,
 *                         1 if it writes the trunk (a stem tensor, or its channel slice of a block output) else 0, its position in
 *                         the forward's launch order (-1 if the walk did not visit all 94 convs)}.
 * ddpm_inception_pack     raw (device fp32, 4-byte aligned) -> packed (ddpm_inception_packed_bytes, 256-byte aligned): BatchNorm
 *                         folded into each conv in fp64 (w gamma / sqrt(var + eps), beta - mean gamma / sqrt(var + eps)), rounded
 *                         once to fp32; the weights are then rounded to TF32.
 * ddpm_inception_forward  x NCHW fp32 [N][3][H][W] (device, 4-byte aligned); resize: bilinear to 299 x 299 first (align_corners
 *                         False); normalize: 2x - 1.  Blocks 0..last_block run; outs[b] (may be null) <- block b NCHW fp32: [N][64][.][.],
 *                         [N][192][.][.], [N][768][.][.], [N][2048][1][1].  pooled (may be null) <- [N][C] global average of block
 *                         last_block (for block 3 the same values as outs[3]).  ws: ddpm_inception_workspace_bytes(N, H, W,
 *                         resize, last_block) bytes, 256-byte aligned; that call refuses (< 0) an input too small for the block.
 * ddpm_inception_conv_run one conv of the network's kind: x NHWC fp32 [N][H][W][Cin rounded up to 4] (16-byte aligned), raw
 *                         weights and BatchNorm vectors as in the state_dict, out channels [c_off, c_off + Cout) of NHWC
 *                         [N][Ho][Wo][C_total] (Cout, c_off, C_total even); scratch: ddpm_inception_conv_scratch_bytes(d).
 * ddpm_inception_pool_run kind 0: 3 x 3 max, stride 2, no padding; 1: 3 x 3 average, stride 1, padding 1, padding not counted;
 *                         2: 3 x 3 max, stride 1, padding 1.  x NHWC [N][H][W][C]; out channels [c_off, c_off + C) of [N][Ho][Wo][C_total].
 * ddpm_inception_input_run the forward's first kernel: x NCHW [N][3][H][W] -> NHWC [N][Ho][Wo][12], Ho = Wo = 299 with resize,
 *                         else H, W: per pixel {x_hi[3], 0, x_lo[3], 0, x_hi[3], 0}, x_hi = x rounded to TF32, x_lo = x - x_hi, which
 *                         the first conv's packed weights {w_hi, w_hi, w_lo} turn into a 3xTF32 product. */
typedef struct {
    int N, H, W, Cin, Cout, kh, kw, stride, ph, pw, c_off, C_total;
    const float* x;
    const float *w, *gamma, *beta, *mean, *var;
    float* out;
    void* scratch;
    long long scratch_bytes;
} ddpm_inception_conv_desc;
int ddpm_inception_num_params(void);
int ddpm_inception_param_info(int i, const char** name, int* ndim, int dims[4], long long* offset);
int ddpm_inception_conv_info(int i, int info[11]);
long long ddpm_inception_packed_bytes(void);
int ddpm_inception_pack(const float* raw, void* packed, void* stream);
long long ddpm_inception_workspace_bytes(int N, int H, int W, int resize, int last_block);
int ddpm_inception_forward(const void* packed, const float* x, int N, int H, int W, int resize, int normalize, int last_block,
                           float* const outs[4], float* pooled, void* ws, long long ws_bytes, void* stream);
long long ddpm_inception_conv_scratch_bytes(const ddpm_inception_conv_desc* d);
int ddpm_inception_conv_run(const ddpm_inception_conv_desc* d, void* stream);
int ddpm_inception_pool_run(int kind, const float* x, int N, int H, int W, int C, float* out, int c_off, int C_total, void* stream);
int ddpm_inception_input_run(const float* x, int N, int H, int W, int resize, int normalize, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Inception Score (Salimans et al., 2016, as the TensorFlow improved-gan/inception_score.py computes it; inception_score.cuh).
 * Stateless and graph-capturable like the forward; every argument is checked before the first launch.
 * ddpm_is_fc_pack         fc_weight (device fp32 [1008][2048], the checkpoint's fc.weight, 4-byte aligned) -> packed
 *                         (ddpm_is_fc_packed_bytes, 256-byte aligned): per class [w_hi | w_hi | w_lo] with w_hi = tf32(w),
 *                         w_lo = tf32(w - w_hi).
 * ddpm_is_logits          logits fp32 [N][1008] (row pitch 1008, 8-byte aligned) = feats . fc_weight^T, no bias; feats fp32 [N]
 *                         rows of pitch ld >= 2048 (the pooled block-3 features).  A 3xTF32 GEMM (f_hi w_hi + f_lo w_hi + f_hi w_lo,
 *                         fp32 accumulation); a row depends on its own features only.  ws: ddpm_is_logits_workspace_bytes(N)
 *                         bytes, 256-byte aligned.
 * ddpm_is_score           logits fp32 [N][C] (row pitch ld >= C), cut in order into `splits` parts, part i = rows
 *                         [i N / splits, (i + 1) N / splits), 1 <= splits <= N.  out (fp64, splits + 1 values): out[i] =
 *                         exp(mean_x sum_y p(y|x) (log p(y|x) - log pbar_i(y))) with p = softmax over all C classes, computed in fp64
 *                         with log p = z - logsumexp(z); out[splits] = status: 0, or 1 when a logit is not finite (then out[i] are
 *                         NaN).  Fixed-order reductions: the same logits give the same bits.  scratch: ddpm_is_score_scratch_bytes(N,
 *                         C, splits) bytes, 16-byte aligned. */
long long ddpm_is_fc_packed_bytes(void);
int ddpm_is_fc_pack(const float* fc_weight, void* packed, void* stream);
long long ddpm_is_logits_workspace_bytes(int N);
int ddpm_is_logits(const void* packed, const float* feats, int N, long long ld, float* logits, void* ws, long long ws_bytes, void* stream);
long long ddpm_is_score_scratch_bytes(int N, int C, int splits);
int ddpm_is_score(const float* logits, int N, int C, long long ld, int splits, double* out, void* scratch, long long bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Kernel Inception Distance (Binkowski et al., 2018; the unbiased polynomial-kernel MMD^2 over subsets; kid.cuh).
 * ddpm_kid  x fp32 [n1] rows of pitch ldx >= d, y fp32 [n2] rows of pitch ldy >= d (device, 4-byte aligned), 1 <= d <= 4096;
 *           idx_host: a HOST array of S * 2 * m int32 indices, per subset s first ix (m rows of x) then iy (m rows of y), each in
 *           range and distinct within its half (checked before any launch, then copied into the scratch on `stream`), 2 <= m <=
 *           min(n1, n2).  With k(a, b) = (gamma a . b + coef0)^degree, 1 <= degree <= 8, out (fp64, S + 3 values):
 *           out[s] = (sum_{i != j} k(x_i, x_j) + sum_{i != j} k(y_i, y_j)) / (m (m - 1)) - 2 sum_{i, j} k(x_i, y_j) / m^2 over the
 *           rows of subset s, out[S] = their mean, out[S + 1] = their population std, out[S + 2] = status: 0, or 1 when a subset's
 *           kernel sum is not finite (a non-finite feature in a drawn row, or an overflow); then out[S] and out[S + 1] are NaN.
 *           Gram entries and sums in fp64 (DMMA), every reduction in a fixed order: the same rows give the same bits.
 *           scratch: ddpm_kid_scratch_bytes(S, m) bytes, 16-byte aligned. */
long long ddpm_kid_scratch_bytes(int S, int m);
int ddpm_kid(const float* x, long long ldx, int n1, const float* y, long long ldy, int n2, int d, const int32_t* idx_host, int S, int m,
             int degree, double gamma, double coef0, double* out, void* scratch, long long bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Low-level operators: GroupNorm(32, C, eps=1e-6) [+ SiLU] [+ dropout] (unet.py:18-20,83-84) and the bias column sums, with the
 * launch geometry the UNet engine's plans use (used by the parity tests of the engine itself).
 * Input = channel concat of two NHWC bf16 sources x0 [B][HW][C0] and x1 [B][HW][C1] (C1 = 0: one source).  C0 and C1 are
 * multiples of 8, C = C0 + C1 is a multiple of 32 and at most 2048.  Arguments are checked before any device work.
 * scratch: caller-owned device area of ddpm_gn_scratch_bytes(B, C) bytes, zeroed by the caller before every call.
 *
 * Forward routes (the engine picks one per norm from the shape):
 *  1  k_gn_stats + k_gn_apply (fp64 group sums)
 *  2  k_gn_small: statistics + apply in one block per image; needs HW <= 64
 *  3  k_gn_apply from the producers' quad statistics qs0 / qs1 [B][C0/4][2] / [B][C1/4][2] fp64 {sum, sum of squares}
 *     (ddpm_gn_epi); needs C % 128 == 0
 *  4  k_gn_prep: K only, from the quad statistics (y is not written); needs C % 128 == 0
 * Outputs: y bf16 [B][HW][C] = act(gn(x)) * keep / (1 - drop_p);  K f32 [B][4][C] = {rstd*gamma, beta - mean*rstd*gamma, rstd,
 * mean*rstd} per (image, channel).  Dropout is on when drop_p > 0 and seed != 0: the keep bit of element (b, p, c) is a Philox
 * draw keyed by (seed, layer) at counter (b*HW + p)*C + c; mask (optional) [B][HW][C/8] receives the keep bits, bit e of byte
 * (b, p, o) = channel 8*o + e. */
typedef struct ddpm_gn_desc {
    int route, B, HW, C0, C1;
    const void* x0; const void* x1;
    const float* gamma; const float* beta;
    int silu; float drop_p; uint64_t seed; uint32_t layer;
    unsigned char* mask;
    const double* qs0; const double* qs1;
    void* y; float* K;
    void* scratch;
} ddpm_gn_desc;
/* Backward of the forward above (autograd of unet.py:83-84 with the saved K and mask): with dn = dy * keep/(1 - drop_p) * act'(y),
 *   dx = rstd*gamma*dn - P*x - Q (+ addend) written to dx0 / dx1 (acc0 / acc1 != 0: added to what is there),
 *   dgamma += sum dn*xhat,  dbeta += sum dn  (over images and pixels).
 * dn_inplace != 0 overwrites dy with bf16(dn) in the first pass.  drop_p > 0 needs the forward's mask.
 * Column sums of dx (any of them may be NULL): cs_per_img[b][cs_ld] +=, cs_total[c] +=, cs_total2[c] +=. */
typedef struct ddpm_gn_bwd_desc {
    int B, HW, C0, C1;
    const void* x0; const void* x1;
    void* dy;
    const float* K; const float* gamma;
    float* dgamma; float* dbeta;
    void* dx0; void* dx1; int acc0, acc1;
    const void* addend;
    int silu; float drop_p; const unsigned char* mask;
    int dn_inplace;
    float* cs_per_img; int cs_ld; float* cs_total; float* cs_total2;
    void* scratch;
} ddpm_gn_bwd_desc;
long long ddpm_gn_scratch_bytes(int B, int C);
int ddpm_groupnorm_fwd_run(const ddpm_gn_desc* d, void* stream);
int ddpm_groupnorm_bwd_run(const ddpm_gn_bwd_desc* d, void* stream);
/* Bias gradients (autograd of the conv / linear bias): column sums of dy bf16 [B][HW][C] over its first C_valid channels,
 * per_img[b][ld] += (optional), total[c] += (optional), total2[c] += (optional).  C a multiple of 8, any width. */
int ddpm_colsum_run(const void* dy, float* per_img, int ld, float* total, float* total2, int B, int HW, int C, int C_valid, void* stream);

/* ------------------------------------------------------------------------------------------------
 * UNet engine.  replaces: UNet.__init__/forward (ddpm_torch/models/unet.py:96-233), its autograd backward,
 * and the model-side half of GaussianDiffusion.train_losses / p_sample_step (diffusion.py:107-158,217-243).
 */
typedef struct ddpm_unet_cfg {          /* mirrors UNet(in_channels, hid_channels, out_channels, ch_multipliers,   */
    int in_channels, hid_channels, out_channels;   /* num_res_blocks, apply_attn, time_embedding_dim, drop_rate)  unet.py:96-107 */
    int levels; int ch_mult[8];
    int num_res_blocks; int attn[8];
    int temb_dim;                       /* 0 -> 4*hid_channels (unet.py:112) */
    float drop_rate;
} ddpm_unet_cfg;
typedef struct ddpm_unet ddpm_unet;

/* ddpm_unet_create(cfg, out) is ddpm_unet_create_ex(cfg, 1, out).  resample_with_conv (unet.py:106,164-170,199-202):
 * 1 = SamePad2d(3, 2) + stride-2 3x3 conv down, nearest x2 + 3x3 conv up;  0 = AvgPool2d(2) down, bare nearest x2 up, and the
 * resample convs are absent from the parameter inventory.  Any other value is refused before anything is allocated. */
int  ddpm_unet_create(const ddpm_unet_cfg* cfg, ddpm_unet** out);
int  ddpm_unet_create_ex(const ddpm_unet_cfg* cfg, int resample_with_conv, ddpm_unet** out);
void ddpm_unet_destroy(ddpm_unet* h);
/* Parameter inventory in the reference's state_dict order (unet.py registration order). Offsets (in fp32 elements)
 * address the FLAT parameter / gradient buffers the caller owns; each tensor is OIHW / [out,in] fp32 as in the reference. */
int       ddpm_unet_num_params(const ddpm_unet* h);
int       ddpm_unet_param_info(const ddpm_unet* h, int i, const char** name, int* ndim, int dims[4], long long* offset);
long long ddpm_unet_flat_elems(const ddpm_unet* h);
/* Graph validity: a CUDA graph captured from this handle's launches stays valid while the value returned here is unchanged.
 * It moves on every ddpm_unet_workspace_bytes and ddpm_unet_plan call (both rebuild the launch lists) and whenever
 * ddpm_sampler_setup or ddpm_bpd_setup reallocates its table for a new length; a setup with the same length rewrites the table
 * in place and leaves it unchanged.  A null handle returns a negative error code. */
long long ddpm_unet_graph_epoch(const ddpm_unet* h);
/* Workspace bytes for a (batch, H, W) plan; training != 0 also plans the backward pass. */
long long ddpm_unet_workspace_bytes(ddpm_unet* h, int B, int H, int W, int training);
/* Bind caller-owned device buffers and compile the launch plan. grads_flat may be NULL when training == 0. */
int ddpm_unet_plan(ddpm_unet* h, int B, int H, int W, int training, float* params_flat, float* grads_flat,
                   void* workspace, long long workspace_bytes);
/* Re-pack fp32 master weights into the bf16 kernel layouts; call after every parameter update / load_state_dict.
 * Ordered after everything queued on `stream` so far.  For a TRAINING plan the pack kernels run on the engine's internal stream
 * and the next forward/train_forward call joins them right before its first packed-weight consumer, so the pack overlaps the
 * timestep-embedding MLP and q_sample + in_conv of that forward; inference plans pack in `stream`. */
int ddpm_unet_repack(ddpm_unet* h, void* stream);
/* eps = UNet(x, t):  x f32[B,Cin,H,W] NCHW, t i64[B], eps f32[B,Cout,H,W]   (unet.py:205-233) */
int ddpm_unet_forward(ddpm_unet* h, const float* x, const int64_t* t, float* eps, uint64_t dropout_seed, void* stream);
/* Backward of the last forward: d_eps f32[B,Cout,H,W] -> flat grads (zeroed then written). x,t must be unchanged.
 * Same as ddpm_unet_backward_ex(h, d_eps, NULL, 1, stream). */
int ddpm_unet_backward(ddpm_unet* h, const float* d_eps, void* stream);
/* Backward of the last forward with a choice of outputs (autograd of unet.py:205-233 with respect to x and/or the parameters):
 *  dx           f32[B,Cin,H,W] NCHW <- d(eps . d_eps)/dx, the gradient with respect to the network input (guided sampling,
 *               inverse problems, saliency); NULL = not computed.
 *  param_grads  1: the flat gradients are zeroed and then written, as ddpm_unet_backward does;
 *               0: no weight-gradient op runs and the flat gradient buffer is neither read nor written (a frozen model whose
 *               caller may be accumulating gradients of another backward in it).  No gradient-chunk event is recorded:
 *               ddpm_unet_wait_grad_chunk then fails until the next backward with parameter gradients.
 * Refused before any launch without a training plan, when param_grads is not 0 or 1, or when param_grads = 0 and dx = NULL.
 * CUDA-graph capturable. */
int ddpm_unet_backward_ex(ddpm_unet* h, const float* d_eps, float* dx, int param_grads, void* stream);
/* Kernel launches of one backward of the compiled (or dry-planned) training plan in the variant (want_dx, param_grads), flags
 * 0 or 1 and not both 0 (memsets not counted); (0, 1) is the backward of ddpm_unet_launch_counts.  < 0 on error. */
int ddpm_unet_backward_launches(const ddpm_unet* h, int want_dx, int param_grads);
/* Fused training forward (diffusion.py:217-243, mse/eps branch): x_t = q_sample(x0,t,noise) with the fp32 tables
 * tab_sqrt_ab / tab_sqrt_1mab [T]; eps = UNet(x_t,t); losses[b] = mean((noise-eps)^2).
 * Needs out_channels == in_channels (fails before any launch otherwise), as do the sampler steps below. */
int ddpm_train_forward(ddpm_unet* h, const float* x0, const int64_t* t, const float* noise, const float* tab_sqrt_ab,
                       const float* tab_sqrt_1mab, float* losses, uint64_t dropout_seed, void* stream);
/* Backward of ddpm_train_forward given d(sum)/d(losses[b]) = gscale[b] (f32[B]). */
int ddpm_train_backward(ddpm_unet* h, const float* gscale, void* stream);
/* Sampler (diffusion.py:152-174, ddim.py:96-113).  setup uploads per-step tables: t_model[S] (timestep fed to the UNet),
 * coef[S][6] = {sqrt_recip_ab, sqrt_recip_m1_ab, post_c1, post_c2, exp(.5*logvar), t>0}; both HOST pointers.
 * reset(step) arms the device-side step counter; each step() call then consumes one step (counter decrements),
 * x f32[B,C,H,W] is updated in place; z = per-step N(0,1) draw (device) or NULL (+seed != 0: built-in Philox stream).
 * A step() is a fixed launch sequence with no host-side arguments that change -> capturable once, replayable T times.
 * The alpha/beta update runs in the epilogue of the UNet's final conv (eps never reaches memory; no tail launch). */
int ddpm_sampler_setup(ddpm_unet* h, int S, const int64_t* t_model_host, const float* coef_host);
int ddpm_sampler_reset(ddpm_unet* h, int first_step, void* stream);
int ddpm_sampler_step(ddpm_unet* h, float* x, const float* z, uint64_t seed, void* stream);
/* Same step, additionally writing the clipped x_0 prediction of diffusion.py:122,130 to pred_x0 f32[B,C,H,W] (NULL = skip):
 * GaussianDiffusion.p_sample_progressive (diffusion.py:176-198, p_sample_step(..., return_pred=True)). */
int ddpm_sampler_step_pred(ddpm_unet* h, float* x, const float* z, uint64_t seed, float* pred_x0, void* stream);
/* Log-likelihood in bits per dimension: one timestep of GaussianDiffusion.calc_all_bpd (diffusion.py:252-268) with its
 * _loss_term_bpd (:203-215), eps-prediction and fixed variance.
 * setup uploads the per-step rows coef[T][9] = {sqrt_ab, sqrt_1mab, sqrt_recip_ab, sqrt_recip_m1_ab, post_c1, post_c2,
 * model_logvar, true_logvar, t>0} (HOST pointer; fp32 values cast from the fp64 tables as _extract does, diffusion.py:83).
 * The table is owned by the handle, kept apart from the sampler's, and re-used when T is unchanged.
 * reset(step) arms the device-side step counter (shared with the sampler); each step() call consumes one step ti (counter
 * decrements): x_t = q_sample(x0, ti, noise) (diffusion.py:92-97) formed in in_conv's loads, eps = UNet(x_t, ti), then in the
 * epilogue of the final conv (a tail kernel on plans whose out_conv is not on the tensor cores):
 *   losses[b][ti] = mean_{c,y,x}(t > 0 ? KL(q(x_{t-1}|x_t,x_0) || p(x_{t-1}|x_t)) : -log p(x_0|x_1)) / ln 2
 *   mses[b][ti]   = mean_{c,y,x}((pred_x0 - x0)^2),  pred_x0 clamped to [-1, 1] when clip_denoised != 0
 * x0, noise f32[B,C,H,W]; losses, mses f32[B][T].  Per-block partial sums and a fixed-order finalise: no floating-point atomics.
 * A step() is a fixed launch sequence with no host-side arguments that change -> capturable once, replayable T times. */
int ddpm_bpd_setup(ddpm_unet* h, int T, const float* coef_host);
int ddpm_bpd_reset(ddpm_unet* h, int first_step, void* stream);
int ddpm_bpd_step(ddpm_unet* h, const float* x0, const float* noise, int clip_denoised, float* losses, float* mses, void* stream);
/* Data-parallel training (train.py:110 DDP, utils/train.py:149-153): the backward pass finishes the flat gradient buffer in
 * contiguous CHUNKS, level group by level group, and records a CUDA event per chunk.  grad_chunks returns their number and
 * fills lo/hi (element offsets into the flat buffer, in completion order; together they tile it exactly); wait_grad_chunk makes
 * `stream` wait for chunk i of the most recent ddpm_unet_backward / ddpm_train_backward, so that the caller can all-reduce that
 * chunk on a communication stream while the rest of the backward is still running.  Needs a training plan. */
int ddpm_unet_grad_chunks(const ddpm_unet* h, int max_n, long long* lo, long long* hi);
int ddpm_unet_wait_grad_chunk(ddpm_unet* h, int i, void* stream);
/* Introspection for tests / bench: op counts and algorithmic FLOPs of the compiled plan. */
int ddpm_unet_plan_stats(const ddpm_unet* h, int* n_fwd_ops, int* n_bwd_ops, int* n_tensorcore_ops, int* n_generic_ops,
                         double* fwd_flops, double* bwd_flops);
int ddpm_unet_launches_per_forward(const ddpm_unet* h);
/* kernel launches issued by one forward / backward / repack of the compiled plan (memsets not counted) */
int ddpm_unet_launch_counts(const ddpm_unet* h, int* fwd, int* bwd, int* pack);

/* ---- timestep-path probes: run a plan's own timestep ops alone (operator-level tests of the engine).
 * Layout of a planned (or dry-planned) handle's per-block projections TP [B][tp_ld]: route 0 = CUDA cores, 1 = tensor cores;
 * has_uniform = the plan has the one-row route ddpm_sampler_step swaps in; block i (in the order the forward runs the ResBlocks,
 * e.g. "downsamples.level_1.0.0") owns columns off[i] .. off[i] + cout[i] - 1 of TP, the output of its `fc`.  Fills at most max_n
 * entries of off / cout / block (any pointer may be NULL; the names live until the next plan) and returns the block count. */
int ddpm_unet_temb_layout(const ddpm_unet* h, int max_n, int* route, int* has_uniform, int* temb_dim, int* tp_ld, int* maxc,
                          int* off, int* cout, const char** block);
/* The plan's "zero.fwd" op, then its timestep ops (uniform = 1: the one-row ops + broadcast exactly as ddpm_sampler_step runs
 * them; refused on a plan without them), waiting for a pending repack as the forward does.  Copies out (device pointers, any may
 * be NULL) emb [B][hid], e0 = Linear(emb) [B][E], e1 = Linear(SiLU(e0)) [B][E] (row 0 only under uniform) and TP [B][tp_ld]. */
int ddpm_unet_temb_forward(ddpm_unet* h, const int64_t* t, int uniform, float* emb, float* e0, float* e1, float* tp, void* stream);
/* Training plans, right after a per-row ddpm_unet_temb_forward (any other forward of the plan in between is refused): the backward's "zero.bwd" op (which clears the flat gradient buffer),
 * dtp [B][tp_ld] (device) copied into the plan's dTP, then the backward's timestep ops; the fc.weight and embed.* gradients land
 * in the flat gradient buffer.  Copies out d_st = dL/dSiLU(e1) and d_s0 = dL/dSiLU(e0), [B][E] each (may be NULL). */
int ddpm_unet_temb_backward(ddpm_unet* h, const float* dtp, float* d_st, float* d_s0, void* stream);

/* ---- image-side convolution probes: run a plan's own in_conv and out_conv.2 ops alone (operator-level tests of the engine).
 * Routes of a planned (or dry-planned) handle, 1 = tensor cores, 0 = CUDA cores, -1 = not in this plan (an inference plan has no
 * weight gradient and no dx): in_conv forward, in_conv weight gradient, out_conv.2 (forward and backward) and the input gradient
 * dx; h0_qstats = 1 when in_conv writes h0's GroupNorm quad statistics [B][hid/4][2] fp64 {sum, sum of squares}.  Any pointer may
 * be NULL. */
int ddpm_unet_image_layout(const ddpm_unet* h, int* in_route, int* in_wgrad_route, int* out_route, int* dx_route, int* h0_qstats);
/* The plan's "zero.fwd" op and its in_conv ops over x [B][Cin][H][W] fp32 (with noise set, the q_sample prologue forms
 * x_t = tab_a[t_b]*x + tab_s[t_b]*noise as ddpm_train_forward does; noise needs t and both tables); then a [B][H][W][hid] bf16
 * (device) copied into out_conv.0's output and the plan's out_conv.2 ops, eps_out [B][Cout][H][W] fp32, waiting for a pending
 * repack as the forward does.  Copies out (device pointers, may be NULL) x_t [B][Cin][H][W] fp32 (needs noise), h0 [B][H][W][hid]
 * bf16 and its quad statistics (refused on a plan without them).  x must stay valid until the matching backward. */
int ddpm_unet_image_forward(ddpm_unet* h, const float* x, const int64_t* t, const float* noise, const float* tab_a, const float* tab_s,
                            const void* a, float* xt_out, void* h0_out, double* h0_qstats_out, float* eps_out, void* stream);
/* Training plans, right after a ddpm_unet_image_forward (any other forward of the plan in between is refused): the backward's
 * "zero.bwd" op (which clears the flat gradient buffer), out_conv.2's backward ops over d_eps [B][Cout][H][W] fp32, then dh0
 * [B][H][W][hid] bf16 (device) copied into the plan's gradient of h0 and in_conv's backward ops (with dx_out set, the input-gradient
 * ops too: dx_out [B][Cin][H][W] fp32).  The in_conv.* and out_conv.2.* gradients land in the flat gradient buffer; d_a_out
 * [B][H][W][hid] bf16 (may be NULL) receives the gradient of out_conv.0's output. */
int ddpm_unet_image_backward(ddpm_unet* h, const float* d_eps, const void* dh0, float* dx_out, void* d_a_out, void* stream);

/* ---- fused optimizer step over the flat fp32 buffers.
 * Replaces, per training step, nn.utils.clip_grad_norm_(params, max_norm) + Adam.step() + LambdaLR warm-up + EMA.update()
 * (utils/train.py:159-165, :300-305; train.py:128-132) = ~13 tiny kernels x 304 tensors, by two launches and no host sync.
 *   step          : 1-based Adam step t (bias corrections 1 - beta^t), lr is the already-scheduled learning rate of this step
 *   max_grad_norm : <= 0 disables clipping;  ema_decay : < 0 disables the EMA update (ema_shadow may then be NULL);
 *   ema_num_updates: 0-based n of utils/train.py:301-302, decay_t = min(ema_decay, (1 + n) / (10 + n))
 *   state         : device scratch of >= 64 bytes, zero-initialised ONCE by the caller (fp64 accumulator + ticket)
 *   norm_out      : device float[2] <- {total_norm before clipping, clip coefficient applied}
 * n (elements) must be a multiple of 4 and all buffers 16-byte aligned (the flat layout guarantees both). */
typedef struct ddpm_opt_cfg {
  double lr, beta1, beta2, eps, max_grad_norm, ema_decay;
  int step, ema_num_updates;
} ddpm_opt_cfg;
int ddpm_opt_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, float* ema_shadow, long long n,
                  const ddpm_opt_cfg* cfg, void* state, float* norm_out, void* stream);

/* ---- generate.py:129 post-processing on the device:
 * out[b][y][x][c] = uint8(clamp(round(x[b][c][y][x] * 127.5 + 127.5), 0, 255)) - NCHW fp32 samples -> NHWC uint8 images, the
 * layout PIL.Image.fromarray consumes (generate.py:112-114).  Bit-exact with the reference expression.  C in 1..4. */
int ddpm_to_uint8_nhwc(const float* x, uint8_t* out, int B, int C, int H, int W, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2-D toy denoiser (ddpm_torch/toy/toy_model.py: Decoder(in_features, mid_features, num_temporal_layers)) on wgmma (toy_mlp.cuh).
 * Stateless: every call takes the configuration and the current fp32 parameter pointers (device, in the reference's parameters()
 * order; the four [M][M] weights 16-byte aligned), so updates by any optimiser or p.data.copy_ are seen without a repack.
 * Supported: mid_features M in {64, 128}, in_features D in 1..4, num_layers L >= 1, B >= 1; anything else is refused before any
 * launch.  No allocation, no synchronisation, graph-capturable; the caller's stream.
 * ws: caller-owned device workspace of ddpm_toy_workspace_bytes(cfg, rows, training) bytes, 256-byte aligned.  A training forward
 * fills it with what the matching backward reads, so it must be kept until that backward has run.
 * ddpm_toy_forward        x f32 [B][D], t i64 [B] -> out f32 [B][D]; training != 0 saves the activations for ddpm_toy_backward
 * ddpm_toy_train_forward  losses[b] = mean((noise - Decoder(q_sample(x0, t, noise), t))^2) with sqrt_ab / sqrt_1mab f32 [T] (always
 *                         saves; workspace with training = 1)
 * ddpm_toy_backward       d_out f32 [B][D] -> grad f32 [P] (flat, parameters() order, overwritten) and dx f32 [B][D] (optional)
 * ddpm_toy_train_backward per-row loss gradient g f32 [B] (and the same noise) -> grad
 * ddpm_toy_sample         the whole p_sample chain (toy/diffusion.py: no clip) in one launch after the step table: x f32 [B][D] in
 *                         place, coef f32 [S][6] = {sqrt_recip_ab, sqrt_recip_m1_ab, coef1, coef2, sigma, t > 0}, z f32 [S][B][D]
 *                         (z[k] at t = S-1-k); workspace ddpm_toy_workspace_bytes(cfg, S, 0)
 * Gradients are summed in a fixed order (per-CTA partials, then one reduce): a training step is bit-reproducible. */
typedef struct { int in_features, mid_features, num_layers; } ddpm_toy_cfg;
typedef struct {
    const float *in_fc_weight, *norm1_weight, *norm1_bias, *fc1_weight, *norm2_weight, *norm2_bias, *fc2_weight, *enc_weight,
        *enc_bias, *out_norm_weight, *out_norm_bias, *out_fc_weight, *out_fc_bias, *t_proj_weight, *t_proj_bias;
} ddpm_toy_params;
long long ddpm_toy_num_params(const ddpm_toy_cfg* cfg);
long long ddpm_toy_workspace_bytes(const ddpm_toy_cfg* cfg, long long rows, int training);
int ddpm_toy_forward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const float* x, const long long* t, long long B, float* out,
                     int training, void* ws, long long ws_bytes, void* stream);
int ddpm_toy_train_forward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const float* x0, const long long* t, const float* noise,
                           const float* sqrt_ab, const float* sqrt_1mab, long long B, float* losses, void* ws, long long ws_bytes,
                           void* stream);
int ddpm_toy_backward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const long long* t, const float* d_out, long long B,
                      float* dx, float* grad, void* ws, long long ws_bytes, void* stream);
int ddpm_toy_train_backward(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, const long long* t, const float* noise, const float* g,
                            long long B, float* grad, void* ws, long long ws_bytes, void* stream);
int ddpm_toy_sample(const ddpm_toy_cfg* cfg, const ddpm_toy_params* p, float* x, long long B, int S, const float* coef,
                    const float* z, void* ws, long long ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DDPM_B200_H */
