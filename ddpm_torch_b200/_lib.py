"""ctypes binding of libddpm_b200.so (the C ABI declared in include/ddpm_b200.h).

The extension is built in-tree by ``__graft_entry__.build()`` / ``csrc/build.sh``.  There is NO fallback:
if the shared library is missing or the device is not sm_90, every entry point raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libddpm_b200.so")


class GnEpi(C.Structure):
    _fields_ = [("qstats", C.c_void_p)]


class GemmDesc(C.Structure):
    _fields_ = [
        ("mode", C.c_int), ("block_n", C.c_int), ("M", C.c_int), ("N", C.c_int),
        ("W", C.c_int), ("H", C.c_int), ("NB", C.c_int),
        ("a_ptr", C.c_void_p * 3), ("a_C", C.c_int * 3), ("a_ld", C.c_longlong * 3),
        ("nseg", C.c_int), ("seg_map", C.c_int * 3), ("seg_taps", C.c_int * 3),
        ("seg_kchunks", C.c_int * 3), ("seg_cbase", C.c_int * 3),
        ("b_ptr", C.c_void_p), ("b_K", C.c_int), ("b_rows", C.c_int), ("b_batch", C.c_int),
        ("b_ld", C.c_longlong), ("b_bs", C.c_longlong),
        ("b_k_base", C.c_int), ("a_z_n", C.c_int), ("b_z", C.c_int),
        ("taps", C.c_int), ("splits", C.c_int), ("kblocks", C.c_int),
        ("a_c_base", C.c_int), ("b_c_base", C.c_int), ("grid_z", C.c_int),
        ("out", C.c_void_p), ("ldo", C.c_int), ("out_z_stride", C.c_longlong),
        ("out_tap_stride", C.c_longlong), ("flags", C.c_int),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_ld", C.c_int), ("rows_per_vec", C.c_int),
        ("residual", C.c_void_p), ("ldr", C.c_int), ("alpha", C.c_float),
        ("a_estride", C.c_int), ("b_estride", C.c_int), ("b_pad", C.c_int),
        ("seg_custom", C.c_int * 3), ("seg_cmul", C.c_int * 3),
        ("seg_dx", (C.c_byte * 9) * 3), ("seg_dy", (C.c_byte * 9) * 3),
        ("o_mul", C.c_int), ("o_py", C.c_int), ("o_px", C.c_int), ("kk_splits", C.c_int),
        ("gn", GnEpi), ("cta_pair", C.c_int),
    ]


class HaloDesc(C.Structure):
    _fields_ = [
        ("NB", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cout", C.c_int),
        ("a_ptr", C.c_void_p * 3), ("a_C", C.c_int * 3), ("a_ld", C.c_longlong * 3),
        ("nseg", C.c_int), ("seg_map", C.c_int * 3), ("seg_taps", C.c_int * 3), ("seg_kchunks", C.c_int * 3), ("seg_cbase", C.c_int * 3),
        ("w", C.c_void_p), ("ldw", C.c_longlong), ("Ktot", C.c_int),
        ("out", C.c_void_p), ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_ld", C.c_int), ("residual", C.c_void_p),
        ("base_offset_mode", C.c_int), ("force_sub", C.c_int),
        ("gn", GnEpi), ("xf_K", C.c_void_p), ("xf_silu", C.c_int),
    ]


class GnDesc(C.Structure):
    _fields_ = [
        ("route", C.c_int), ("B", C.c_int), ("HW", C.c_int), ("C0", C.c_int), ("C1", C.c_int),
        ("x0", C.c_void_p), ("x1", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("silu", C.c_int), ("drop_p", C.c_float), ("seed", C.c_uint64), ("layer", C.c_uint32),
        ("mask", C.c_void_p), ("qs0", C.c_void_p), ("qs1", C.c_void_p),
        ("y", C.c_void_p), ("K", C.c_void_p), ("scratch", C.c_void_p),
    ]


class GnBwdDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("HW", C.c_int), ("C0", C.c_int), ("C1", C.c_int),
        ("x0", C.c_void_p), ("x1", C.c_void_p), ("dy", C.c_void_p), ("K", C.c_void_p), ("gamma", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
        ("dx0", C.c_void_p), ("dx1", C.c_void_p), ("acc0", C.c_int), ("acc1", C.c_int),
        ("addend", C.c_void_p),
        ("silu", C.c_int), ("drop_p", C.c_float), ("mask", C.c_void_p),
        ("dn_inplace", C.c_int),
        ("cs_per_img", C.c_void_p), ("cs_ld", C.c_int), ("cs_total", C.c_void_p), ("cs_total2", C.c_void_p),
        ("scratch", C.c_void_p),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("route", C.c_int), ("NB", C.c_int), ("T", C.c_int), ("C", C.c_int),
        ("qkv", C.c_void_p), ("out", C.c_void_p), ("probs", C.c_void_p), ("scratch", C.c_void_p),
    ]


class AttnBwdDesc(C.Structure):
    _fields_ = [
        ("route", C.c_int), ("NB", C.c_int), ("T", C.c_int), ("C", C.c_int),
        ("qkv", C.c_void_p), ("d_out", C.c_void_p), ("probs", C.c_void_p),
        ("d_qkv", C.c_void_p), ("d_scores", C.c_void_p), ("scratch", C.c_void_p),
    ]


class ConvReport(C.Structure):
    _fields_ = [("route", C.c_int), ("launches", C.c_int), ("block_n", C.c_int), ("splits", C.c_int), ("zero_bytes", C.c_longlong)]


class ConvDesc(C.Structure):
    _fields_ = [
        ("op", C.c_int), ("route", C.c_int),
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("ksize", C.c_int), ("stride", C.c_int), ("upsample", C.c_int),
        ("Cin0", C.c_int), ("Cin1", C.c_int), ("Co", C.c_int), ("Cs0", C.c_int), ("Cs1", C.c_int), ("identity_skip", C.c_int),
        ("x0", C.c_void_p), ("x1", C.c_void_p), ("s0", C.c_void_p), ("s1", C.c_void_p), ("dy", C.c_void_p),
        ("w", C.c_void_p), ("w_skip", C.c_void_p),
        ("bias", C.c_void_p), ("skip_bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_ld", C.c_int),
        ("residual", C.c_void_p), ("accumulate", C.c_int),
        ("out", C.c_void_p), ("qstats", C.c_void_p),
        ("scratch", C.c_void_p),
        ("dry", C.c_int),
        ("report", C.POINTER(ConvReport)),
    ]


class IncConvDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("N", "H", "W", "Cin", "Cout", "kh", "kw", "stride", "ph", "pw", "c_off", "C_total")] + [
        ("x", C.c_void_p), ("w", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("mean", C.c_void_p), ("var", C.c_void_p),
        ("out", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_longlong)]


class UnetCfg(C.Structure):
    _fields_ = [("in_channels", C.c_int), ("hid_channels", C.c_int), ("out_channels", C.c_int),
                ("levels", C.c_int), ("ch_mult", C.c_int * 8), ("num_res_blocks", C.c_int), ("attn", C.c_int * 8),
                ("temb_dim", C.c_int), ("drop_rate", C.c_float)]


class OptCfg(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("max_grad_norm", C.c_double), ("ema_decay", C.c_double), ("step", C.c_int), ("ema_num_updates", C.c_int)]


_lib = None


def lib():
    """Load the shared library once.  Raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not built — run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(ddpm_torch_b200 has no CPU/PyTorch fallback)")
        L = C.CDLL(LIB_PATH)
        L.ddpm_last_error.restype = C.c_char_p
        L.ddpm_runtime_check.restype = C.c_int
        L.ddpm_device_error_flag.restype = C.c_int
        L.ddpm_gemm_run.argtypes = [C.POINTER(GemmDesc), C.c_void_p]
        L.ddpm_gemm_run.restype = C.c_int
        vp, i32, i64, u64 = C.c_void_p, C.c_int, C.c_longlong, C.c_uint64
        sig = {
            "ddpm_conv_halo_run": ([C.POINTER(HaloDesc), vp], i32),
            "ddpm_attn_fused_run": ([vp, vp, vp, i32, i32, i32, vp], i32),
            "ddpm_attn_fused_bwd_run": ([vp, vp, vp, vp, vp, i32, i32, i32, vp], i32),
            "ddpm_attention_fwd_run": ([C.POINTER(AttnDesc), vp], i32),
            "ddpm_attention_bwd_run": ([C.POINTER(AttnBwdDesc), vp], i32),
            "ddpm_attn_scratch_bytes": ([i32, i32, i32, i32, i32], i64),
            "ddpm_conv_run": ([C.POINTER(ConvDesc), vp], i32),
            "ddpm_conv_scratch_bytes": ([C.POINTER(ConvDesc)], i64),
            "ddpm_gn_scratch_bytes": ([i32, i32], i64),
            "ddpm_groupnorm_fwd_run": ([C.POINTER(GnDesc), vp], i32),
            "ddpm_groupnorm_bwd_run": ([C.POINTER(GnBwdDesc), vp], i32),
            "ddpm_colsum_run": ([vp, vp, i32, vp, vp, i32, i32, i32, i32, vp], i32),
            "ddpm_unet_create": ([C.POINTER(UnetCfg), C.POINTER(vp)], i32),
            "ddpm_unet_create_ex": ([C.POINTER(UnetCfg), i32, C.POINTER(vp)], i32),
            "ddpm_unet_destroy": ([vp], None),
            "ddpm_unet_num_params": ([vp], i32),
            "ddpm_unet_param_info": ([vp, i32, C.POINTER(C.c_char_p), C.POINTER(i32), C.POINTER(i32 * 4), C.POINTER(i64)], i32),
            "ddpm_unet_flat_elems": ([vp], i64),
            "ddpm_unet_graph_epoch": ([vp], i64),
            "ddpm_unet_workspace_bytes": ([vp, i32, i32, i32, i32], i64),
            "ddpm_unet_plan": ([vp, i32, i32, i32, i32, vp, vp, vp, i64], i32),
            "ddpm_unet_repack": ([vp, vp], i32),
            "ddpm_unet_forward": ([vp, vp, vp, vp, u64, vp], i32),
            "ddpm_unet_backward": ([vp, vp, vp], i32),
            "ddpm_unet_backward_ex": ([vp, vp, vp, i32, vp], i32),
            "ddpm_unet_backward_launches": ([vp, i32, i32], i32),
            "ddpm_train_forward": ([vp, vp, vp, vp, vp, vp, vp, u64, vp], i32),
            "ddpm_train_backward": ([vp, vp, vp], i32),
            "ddpm_sampler_setup": ([vp, i32, vp, vp], i32),
            "ddpm_sampler_reset": ([vp, i32, vp], i32),
            "ddpm_sampler_step": ([vp, vp, vp, u64, vp], i32),
            "ddpm_sampler_step_pred": ([vp, vp, vp, u64, vp, vp], i32),
            "ddpm_bpd_setup": ([vp, i32, vp], i32),
            "ddpm_bpd_reset": ([vp, i32, vp], i32),
            "ddpm_bpd_step": ([vp, vp, vp, i32, vp, vp, vp], i32),
            "ddpm_unet_grad_chunks": ([vp, i32, C.POINTER(i64), C.POINTER(i64)], i32),
            "ddpm_unet_wait_grad_chunk": ([vp, i32, vp], i32),
            "ddpm_unet_plan_stats": ([vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                      C.POINTER(C.c_double), C.POINTER(C.c_double)], i32),
            "ddpm_unet_launches_per_forward": ([vp], i32),
            "ddpm_unet_launch_counts": ([vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)], i32),
            "ddpm_opt_step": ([vp, vp, vp, vp, vp, i64, C.POINTER(OptCfg), vp, vp, vp], i32),
            "ddpm_to_uint8_nhwc": ([vp, vp, i32, i32, i32, i32, vp], i32),
            "ddpm_unet_temb_layout": ([vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                       C.POINTER(i32), C.POINTER(i32), C.POINTER(C.c_char_p)], i32),
            "ddpm_unet_temb_forward": ([vp, vp, i32, vp, vp, vp, vp, vp], i32),
            "ddpm_unet_temb_backward": ([vp, vp, vp, vp, vp], i32),
            "ddpm_unet_image_layout": ([vp] + [C.POINTER(i32)] * 5, i32),
            "ddpm_unet_image_forward": ([vp] * 12, i32),
            "ddpm_unet_image_backward": ([vp] * 6, i32),
            "ddpm_knn_scratch_bytes": ([i32, i32, i32, i32], i64),
            "ddpm_knn_kth": ([vp, i32, i64, vp, i32, i64, i32, i32, vp, vp, i64, vp], i32),
            "ddpm_knn_cover": ([vp, i32, i64, vp, i32, i64, i32, vp, vp, vp, i64, vp], i32),
            "ddpm_fid_stats_bytes": ([i32], i64),
            "ddpm_fid_stats_update": ([vp, i32, vp, i64, i64, vp], i32),
            "ddpm_fid_stats_finalize": ([vp, i32, i64, i32, vp, vp, vp], i32),
            "ddpm_fid_distance_scratch_bytes": ([i32], i64),
            "ddpm_fid_distance": ([vp, vp, vp, vp, i32, vp, vp, i64, vp], i32),
            "ddpm_inception_num_params": ([], i32),
            "ddpm_inception_param_info": ([i32, C.POINTER(C.c_char_p), C.POINTER(i32), C.POINTER(i32 * 4), C.POINTER(i64)], i32),
            "ddpm_inception_conv_info": ([i32, C.POINTER(i32 * 11)], i32),
            "ddpm_inception_packed_bytes": ([], i64),
            "ddpm_inception_pack": ([vp, vp, vp], i32),
            "ddpm_inception_workspace_bytes": ([i32, i32, i32, i32, i32], i64),
            "ddpm_inception_forward": ([vp, vp, i32, i32, i32, i32, i32, i32, C.POINTER(vp * 4), vp, vp, i64, vp], i32),
            "ddpm_inception_conv_scratch_bytes": ([C.POINTER(IncConvDesc)], i64),
            "ddpm_inception_conv_run": ([C.POINTER(IncConvDesc), vp], i32),
            "ddpm_inception_pool_run": ([i32, vp, i32, i32, i32, i32, vp, i32, i32, vp], i32),
            "ddpm_inception_input_run": ([vp, i32, i32, i32, i32, i32, vp, vp], i32),
            "ddpm_is_fc_packed_bytes": ([], i64),
            "ddpm_is_fc_pack": ([vp, vp, vp], i32),
            "ddpm_is_logits_workspace_bytes": ([i32], i64),
            "ddpm_is_logits": ([vp, vp, i32, i64, vp, vp, i64, vp], i32),
            "ddpm_is_score_scratch_bytes": ([i32, i32, i32], i64),
            "ddpm_is_score": ([vp, i32, i32, i64, i32, vp, vp, i64, vp], i32),
            "ddpm_kid_scratch_bytes": ([i32, i32], i64),
            "ddpm_kid": ([vp, i64, i32, vp, i64, i32, i32, vp, i32, i32, i32, C.c_double, C.c_double, vp, vp, i64, vp], i32),
            "ddpm_toy_num_params": ([vp], i64),
            "ddpm_toy_workspace_bytes": ([vp, i64, i32], i64),
            "ddpm_toy_forward": ([vp, vp, vp, vp, i64, vp, i32, vp, i64, vp], i32),
            "ddpm_toy_train_forward": ([vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, i64, vp], i32),
            "ddpm_toy_backward": ([vp, vp, vp, vp, i64, vp, vp, vp, i64, vp], i32),
            "ddpm_toy_train_backward": ([vp, vp, vp, vp, vp, i64, vp, vp, i64, vp], i32),
            "ddpm_toy_sample": ([vp, vp, vp, i64, i32, vp, vp, vp, i64, vp], i32),
        }
        for name, (args, res) in sig.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = res
        _lib = L
    return _lib


EXPORTS = ["ddpm_last_error", "ddpm_runtime_check", "ddpm_device_error_flag", "ddpm_gemm_run", "ddpm_conv_halo_run", "ddpm_attn_fused_run", "ddpm_attn_fused_bwd_run",
           "ddpm_attention_fwd_run", "ddpm_attention_bwd_run", "ddpm_attn_scratch_bytes", "ddpm_conv_run", "ddpm_conv_scratch_bytes",
           "ddpm_gn_scratch_bytes", "ddpm_groupnorm_fwd_run", "ddpm_groupnorm_bwd_run", "ddpm_colsum_run",
           "ddpm_unet_create", "ddpm_unet_create_ex", "ddpm_unet_destroy", "ddpm_unet_num_params", "ddpm_unet_param_info",
           "ddpm_unet_flat_elems", "ddpm_unet_graph_epoch", "ddpm_unet_workspace_bytes", "ddpm_unet_plan", "ddpm_unet_repack",
           "ddpm_unet_forward", "ddpm_unet_backward", "ddpm_unet_backward_ex", "ddpm_unet_backward_launches", "ddpm_train_forward", "ddpm_train_backward",
           "ddpm_sampler_setup", "ddpm_sampler_reset", "ddpm_sampler_step", "ddpm_sampler_step_pred",
           "ddpm_bpd_setup", "ddpm_bpd_reset", "ddpm_bpd_step", "ddpm_unet_grad_chunks", "ddpm_unet_wait_grad_chunk", "ddpm_unet_plan_stats",
           "ddpm_unet_launches_per_forward", "ddpm_unet_launch_counts", "ddpm_opt_step", "ddpm_to_uint8_nhwc",
           "ddpm_unet_temb_layout", "ddpm_unet_temb_forward", "ddpm_unet_temb_backward",
           "ddpm_unet_image_layout", "ddpm_unet_image_forward", "ddpm_unet_image_backward",
           "ddpm_knn_scratch_bytes", "ddpm_knn_kth", "ddpm_knn_cover",
           "ddpm_fid_stats_bytes", "ddpm_fid_stats_update", "ddpm_fid_stats_finalize", "ddpm_fid_distance_scratch_bytes",
           "ddpm_fid_distance", "ddpm_toy_num_params", "ddpm_toy_workspace_bytes", "ddpm_toy_forward", "ddpm_toy_train_forward",
           "ddpm_toy_backward", "ddpm_toy_train_backward", "ddpm_toy_sample",
           "ddpm_inception_num_params", "ddpm_inception_param_info", "ddpm_inception_conv_info", "ddpm_inception_packed_bytes", "ddpm_inception_pack",
           "ddpm_inception_workspace_bytes", "ddpm_inception_forward", "ddpm_inception_conv_scratch_bytes", "ddpm_inception_conv_run",
           "ddpm_inception_pool_run", "ddpm_inception_input_run",
           "ddpm_is_fc_packed_bytes", "ddpm_is_fc_pack", "ddpm_is_logits_workspace_bytes", "ddpm_is_logits",
           "ddpm_is_score_scratch_bytes", "ddpm_is_score", "ddpm_kid_scratch_bytes", "ddpm_kid"]


def check(rc, what=""):
    if rc != 0:
        msg = lib().ddpm_last_error().decode(errors="replace")
        raise RuntimeError(f"ddpm_b200 {what} failed (code {rc}): {msg}")


def runtime_check():
    check(lib().ddpm_runtime_check(), "runtime_check")


def stream_ptr(device=None):
    """Raw handle of torch's current stream ON ``device`` (default: the current device).  Engine calls of a model that
    lives on cuda:N must be issued on cuda:N's stream under a ``torch.cuda.device(N)`` guard (generate.py:59 builds
    ``cuda:{rank}`` models without ever calling set_device)."""
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
