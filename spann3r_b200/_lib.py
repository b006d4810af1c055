"""ctypes binding of libspann3r_b200.so (include/spann3r_b200.h).

This is the ONLY compute backend of the package: if the library is missing or the device is not
an sm_90 (H100) GPU, every op raises -- there is no CPU, eager-PyTorch or Triton fallback.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("S3R_LIB", os.path.join(_HERE, "libspann3r_b200.so"))   # S3R_LIB: A/B an older build

EPI_PLAIN, EPI_PIXSHUF, EPI_QKV, EPI_HEADTAIL = 0, 1, 2, 3
PRECISION_SPLIT, PRECISION_BF16 = 0, 1     # s3r_gemm_desc.precision: three split-bf16 products, or one bf16 product
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float


class GemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", _vp), ("a_lo", _vp), ("b_hi", _vp), ("b_lo", _vp),
        ("groups", _i), ("nb", _i), ("h", _i), ("w", _i), ("kc", _i), ("taps", _i), ("n", _i),
        ("epi", _i), ("act", _i), ("plane_relu", _i), ("force_bn", _i),
        ("bias", _vp),
        ("res1", _vp), ("ldr1", _i64),
        ("res2", _vp), ("ldr2", _i64),
        ("out_f32", _vp), ("ldo", _i64),
        ("out_hi", _vp), ("out_lo", _vp), ("ldp", _i64), ("plane_col0", _i),
        ("ps_s", _i), ("ps_cout", _i),
        ("q_c", _i), ("q_role_base", _i), ("q_ntok", _i), ("q_ntok_pad", _i), ("q_rope", _i), ("q_nb", _i),
        ("q_pos", _vp), ("q_cs", _vp),
        ("q_out", _vp), ("k_out", _vp), ("vt_out", _vp), ("q_scale", _f),
        ("ht_w", _vp), ("ht_b", _vp), ("ht_pts", _vp), ("ht_conf", _vp),
        ("ln_stats", _vp), ("ln_np", _i), ("ln_eps", _f), ("ln_cs", _vp), ("a_swap", _i),
        ("stats_out", _vp),
        ("trace", _vp),
        ("swap_col0", _i), ("k2_out", _vp), ("vt2_out", _vp),
        ("precision", _i),
        ("lda", _i64), ("ldb", _i64), ("b_group_rows", _i64), ("b_static", _i),
    ]


class LossDesc(C.Structure):
    """Mirror of s3r_loss_desc; the pointer arrays are host arrays of device pointers."""
    _fields_ = [
        ("frames", _i), ("batch", _i), ("height", _i), ("width", _i),
        ("norm_mode", _i), ("gt_scale", _i), ("fix_first", _i), ("shift_inv", _i), ("scale_inv", _i), ("conf_loss", _i),
        ("has_dist_clip", _i), ("alpha", _f), ("dist_clip", _f),
        ("pose0", _vp), ("gt_pts", C.POINTER(_vp)), ("valid", C.POINTER(_vp)), ("pred", C.POINTER(_vp)),
        ("conf", C.POINTER(_vp)),
    ]


LOSS_RES_HEADER, LOSS_RES_PER_B = 20, 6


class AttnTrainDesc(C.Structure):
    """Mirror of s3r_attn_train_desc."""
    _fields_ = [
        ("batch", _i), ("heads", _i), ("nq", _i), ("nk", _i), ("dh", _i), ("scale", _f),
        ("q", _vp), ("k", _vp), ("v", _vp),
        ("q_stride", _i64 * 3), ("k_stride", _i64 * 3), ("v_stride", _i64 * 3),
    ]


# ------------------------------------------------------------------------------------------------
# model-level structs of include/spann3r_b200.h (s3r_model_w, s3r_bank): the engine's weights and memory bank
# ------------------------------------------------------------------------------------------------
class Planes(C.Structure):
    _fields_ = [("hi", _vp), ("lo", _vp)]


class LN(C.Structure):
    _fields_ = [("w", _vp), ("b", _vp)]


class Lin(C.Structure):
    _fields_ = [("w", Planes), ("b", _vp), ("cs", _vp), ("cs_hi", _vp)]


class BlockW(C.Structure):
    _fields_ = [("norm1", LN), ("qkv", Lin), ("proj", Lin), ("norm2", LN), ("fc1", Lin), ("fc2", Lin)]


class DecBlockW(C.Structure):
    _fields_ = [("norm1", LN), ("qkv", Lin), ("proj", Lin), ("norm_y", LN), ("norm2", LN), ("q", Lin),
                ("cproj", Lin), ("norm3", LN), ("fc1", Lin), ("fc2", Lin)]


class RcuW(C.Structure):
    _fields_ = [("conv1", Lin), ("conv2", Lin)]


class FusionW(C.Structure):
    _fields_ = [("rcu1", RcuW), ("rcu2", RcuW), ("out_conv", Lin)]


class DptW(C.Structure):
    _fields_ = [("act1_conv", Lin), ("act1_up", Lin), ("act2_conv", Lin), ("act2_up", Lin), ("act3_conv", Lin),
                ("act4_conv", Lin), ("act4_down", Lin), ("layer_rn", Lin * 4), ("refine", FusionW * 4),
                ("head0", Lin), ("head2", Lin), ("head4_w", _vp), ("head4_b", _vp)]


class ModelW(C.Structure):
    _fields_ = [("patch_embed", Lin), ("enc", BlockW * 24), ("enc_norm", LN),
                ("decoder_embed", Lin), ("dec", DecBlockW * 12), ("dec_norm", LN),
                ("key_fc1", Lin), ("key_fc2", Lin), ("dpt", DptW),
                ("pos_patch_embed", Lin), ("val", BlockW * 6), ("value_norm", LN), ("value_out", Lin),
                ("norm_q", LN), ("norm_k", LN), ("norm_v", LN),
                ("rope_cs", _vp), ("rope_maxpos", _i), ("value_dim", _i), ("rope_cs_v", _vp)]


class Bank(C.Structure):
    _fields_ = [("kn_hi", _vp), ("kn_lo", _vp), ("vnt_hi", _vp), ("vnt_lo", _vp), ("k_raw", _vp), ("v_raw", _vp),
                ("attn", _vp), ("count", _vp), ("cap", _i), ("len", _i)]


_PROTOS = {
    "s3r_version": (_i, []),
    "s3r_abi_sizeof": (_i, [_i]),
    "s3r_last_error": (C.c_char_p, []),
    "s3r_device_ok": (_i, []),
    "s3r_split": (_i, [_vp, _i64, _vp, _vp, _i64, _i, _i64, _i, _i, _vp]),
    "s3r_layernorm": (_i, [_vp, _i64, _vp, _vp, _i64, _i64, _f, _i64, _i, _vp, _i64, _vp, _vp, _i64, _i, _i64, _vp]),
    "s3r_rope2d_inplace": (_i, [_vp, _vp, _i64, _i, _i, _i64, _i64, _f, _f, _vp]),
    "s3r_im2col_patch16": (_i, [_vp, _i64, _i64, _i64, _i64, _i, _i, _i, _vp, _vp, _vp]),
    "s3r_im2col_3x3s2": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "s3r_upsample2x": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "s3r_conv_wgrad_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i, _i]),
    "s3r_conv_wgrad": (_i, [_vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _vp, C.c_size_t, _vp, _vp]),
    "s3r_col2im_3x3s2": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "s3r_gemm": (_i, [C.POINTER(GemmDesc), _vp]),
    "s3r_gemm_tile_n": (_i, [C.POINTER(GemmDesc)]),
    "s3r_gemm_plan_bn": (_i, [_i64, _i, _i, _i, _i]),
    "s3r_attention": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i64, _vp]),
    "s3r_conf_score": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "s3r_conf_score_batched": (_i, [_vp, _i, _i64, _vp, _vp, _vp]),
    "s3r_dropout_mask": (_i, [_vp, _i64, C.c_uint64, _f, _vp]),
    "s3r_focal_weiszfeld": (_i, [_vp, _i, _i, _i, _f, _f, _i, _f, _f, _vp, _vp, _vp]),
    "s3r_focal_median": (_i, [_vp, _i, _i, _i, _f, _f, _f, _f, _vp, _vp, _vp]),
    "s3r_pnp_workspace_bytes": (C.c_size_t, [_i, _i]),
    "s3r_pnp_ransac": (_i, [_vp, _vp, _i, _i64, _i, C.c_double, C.c_double, C.c_double, C.c_double, _f, _i, _i, C.c_uint64,
                            _vp, _vp, _vp, _vp]),
    "s3r_pcl_index_bytes": (C.c_size_t, [_i64]),
    "s3r_pcl_index_build": (_i, [_vp, _i, _i64, _vp, _vp, _vp]),
    "s3r_pcl_nearest": (_i, [_vp, _i64, _vp, _i, _i64, _vp, C.c_double, _vp, _vp, _vp]),
    "s3r_pcl_normals": (_i, [_vp, _i64, _i, _vp, _vp]),
    "s3r_pcl_icp_workspace_bytes": (C.c_size_t, []),
    "s3r_pcl_icp": (_i, [_vp, _i, _i64, _vp, _i64, C.c_double, _vp, _i, C.c_double, C.c_double, _vp, _vp, _vp]),
    "s3r_pcl_stats_workspace_bytes": (C.c_size_t, []),
    "s3r_pcl_stats": (_i, [_vp, _i64, C.c_double, _vp, _vp, _vp]),
    "s3r_pcl_abs_dot": (_i, [_vp, _vp, _vp, _i64, _vp, _vp]),
    "s3r_render_workspace_bytes": (C.c_size_t, [_i, _i]),
    "s3r_render_clear": (_i, [_vp, _i, _i, _vp]),
    "s3r_render_splat": (_i, [_vp, _vp, _i64, _i64, _vp, C.c_double, _i, _i, _vp, _vp]),
    "s3r_render_resolve": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "s3r_mesh_grid_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "s3r_mesh_grid_count": (_i, [_vp, _i, _i, _i, _vp, C.c_size_t, _vp, _vp]),
    "s3r_mesh_grid_faces": (_i, [_vp, _vp, _i, _i, _i, _vp, C.c_size_t, _vp, _vp, _vp]),
    "s3r_raster_triangles": (_i, [_vp, _i64, _vp, _i64, _i64, _vp, C.c_double, C.c_double, _i, _i, _vp, _vp]),
    "s3r_raster_resolve": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "s3r_poisson_workspace_bytes": (C.c_size_t, [_i64, _i]),
    "s3r_poisson_offset": (C.c_size_t, [_i64, _i, _i]),
    "s3r_poisson_setup": (_i, [_vp, _vp, _i, _i64, _i, C.c_double, _vp, C.c_size_t, _vp, _vp]),
    "s3r_poisson_solve": (_i, [_i64, _i, C.c_double, _i, _vp, C.c_size_t, _vp, _vp]),
    "s3r_poisson_extract_count": (_i, [_i64, _i, _vp, C.c_size_t, _vp, _vp]),
    "s3r_poisson_extract": (_i, [_i64, _i, _vp, C.c_size_t, _vp, _vp, _vp, _vp]),
    "s3r_pcl_quantile": (_i, [_vp, _i64, C.c_double, _vp, _vp, _vp]),
    "s3r_mesh_compact_workspace_bytes": (C.c_size_t, [_i64, _i64]),
    "s3r_mesh_compact_count": (_i, [_vp, _vp, _i64, _i64, _vp, C.c_size_t, _vp, _vp]),
    "s3r_mesh_compact": (_i, [_vp, _vp, _i64, _i64, _vp, C.c_size_t, _vp, _vp, _vp]),
    "s3r_loss_workspace_bytes": (C.c_size_t, [C.POINTER(LossDesc)]),
    "s3r_loss_forward": (_i, [C.POINTER(LossDesc), _vp, C.c_size_t, _vp, _vp, _vp, _vp, _vp]),
    "s3r_loss_backward": (_i, [C.POINTER(LossDesc), _vp, C.c_size_t, _vp, _vp, _vp, _vp]),
    "s3r_attn_train_workspace_bytes": (C.c_size_t, [C.POINTER(AttnTrainDesc)]),
    "s3r_attn_train_forward": (_i, [C.POINTER(AttnTrainDesc), _vp, _vp, _vp]),
    "s3r_attn_train_backward": (_i, [C.POINTER(AttnTrainDesc), _vp, _vp, _vp, _vp, C.c_size_t, _vp, _vp, _vp, _vp]),
    "s3r_resample_h_u8": (_i, [_vp, _i64, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "s3r_resample_v_u8_norm": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "s3r_views_abi_sizeof": (_i, [_i]),
    "s3r_views_depth": (_i, [_vp, _i, _i64, _vp]),
    "s3r_views_resample_h": (_i, [_vp, _i, _i, _i, _i, _vp]),
    "s3r_views_resample_v_norm": (_i, [_vp, _i, _i, _i, _vp]),
    "s3r_views_resample_v_u8": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "s3r_views_color_jitter": (_i, [_vp, _i, _i64, _vp]),
    "s3r_engine_create": (_vp, [C.POINTER(ModelW), _i, _i, _i, _i]),
    "s3r_engine_create_ex": (_vp, [C.POINTER(ModelW), _i, _i, _i, _i, _i]),
    "s3r_engine_destroy": (None, [_vp]),
    "s3r_engine_encode": (_i, [_vp, _vp, _i, _vp, _vp]),
    "s3r_engine_decode": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "s3r_engine_keyheads": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "s3r_engine_heads": (_i, [_vp, _vp, _vp, _vp]),
    "s3r_engine_value": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "s3r_engine_memory_read": (_i, [_vp, C.POINTER(Bank), _vp, _f, _vp, _vp]),
    "s3r_engine_memory_read_train": (_i, [_vp, C.POINTER(Bank), _vp, _f, _f, C.c_uint64, _vp, _vp]),
    "s3r_engine_memory_append": (_i, [_vp, C.POINTER(Bank), _vp, _vp, _vp]),
    "s3r_engine_check_sim": (_i, [_vp, C.POINTER(Bank), _vp, _i, _vp, _vp]),
    "s3r_engine_memory_read_slots": (_i, [_vp, C.POINTER(Bank), C.POINTER(_i), _vp, _f, _vp, _vp]),
    "s3r_engine_memory_append_slots": (_i, [_vp, C.POINTER(Bank), C.POINTER(_i), C.POINTER(_i), _vp, _vp, _vp]),
    "s3r_engine_check_sim_slots": (_i, [_vp, C.POINTER(Bank), C.POINTER(_i), C.POINTER(_i), _vp, _vp, _vp]),
    "s3r_engine_take_flops": (C.c_double, [_vp]),
    "s3r_engine_take_launches": (C.c_longlong, [_vp]),
    "s3r_engine_profile": (None, [_vp, _i]),
    "s3r_engine_profile_read": (_i, [_vp, C.POINTER(C.c_double)]),
    "s3r_engine_profile_list": (_i, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(_i), _i]),
}


class ViewDepthDesc(C.Structure):
    """Mirror of s3r_view_depth_desc."""
    _fields_ = [
        ("depth", _vp), ("col_src", _vp), ("row_src", _vp),
        ("depthmap", _vp), ("pts3d", _vp), ("valid", _vp), ("nonfinite", _vp),
        ("depth_stride", _i64), ("w", C.c_int32), ("h", C.c_int32), ("transpose", C.c_int32),
        ("intr", _f * 4), ("pose", _f * 12),
    ]


class ViewImageDesc(C.Structure):
    """Mirror of s3r_view_image_desc."""
    _fields_ = [
        ("src", _vp), ("bh", _vp), ("kh", _vp), ("bv", _vp), ("kv", _vp), ("tmp", _vp), ("img", _vp),
        ("row_stride", _i64),
        ("rows", C.c_int32), ("cols", C.c_int32), ("out_rows", C.c_int32), ("ksh", C.c_int32), ("ksv", C.c_int32),
        ("transpose", C.c_int32),
    ]


class ViewJitterDesc(C.Structure):
    """Mirror of s3r_view_jitter_desc."""
    _fields_ = [
        ("u8", _vp), ("img", _vp),
        ("rows", C.c_int32), ("cols", C.c_int32), ("transpose", C.c_int32), ("order", C.c_int32 * 4),
        ("skip", C.c_int32), ("brightness", _f), ("contrast", _f), ("saturation", _f), ("hue_shift", C.c_int32),
    ]

_lib = None


class S3RError(RuntimeError):
    pass


def lib():
    """Load the shared library (once). Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise S3RError(f"{LIB_PATH} not found: run `python -m spann3r_b200.build` "
                           "(the package has no CPU / eager fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def declared_symbols():
    return list(_PROTOS)


def check(status: int, what: str = ""):
    if status != 0:
        msg = lib().s3r_last_error().decode(errors="replace")
        raise S3RError(f"{what} failed with status {status}: {msg}")


def require_device():
    if not torch.cuda.is_available() or not lib().s3r_device_ok():
        raise S3RError("spann3r_b200 needs a CUDA device of compute capability 9.0 (H100); no fallback exists")


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    """Current stream OF THE GIVEN DEVICE (default: the current device).  Callers that take tensors pass the tensor's
    device and run under `on_device(...)`: the library allocates, configures and launches on the CURRENT device."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def on_device(t_or_dev):
    """Context manager: make the tensor's (or given) CUDA device current for the duration of a library call, so that
    `Spann3R(...).to('cuda:1')` works without a global `torch.cuda.set_device(1)` (as the reference's `.to(device)` does)."""
    dev = t_or_dev.device if isinstance(t_or_dev, torch.Tensor) else torch.device(t_or_dev)
    return torch.cuda.device(dev)


def call(name, device, *args):
    """Call library function `name` with `args` and the current stream of `device` appended, with `device` current
    (a tensor, a torch.device, or None for the current device); raise S3RError naming `name` on a nonzero status."""
    dev = device.device if isinstance(device, torch.Tensor) else device
    with torch.cuda.device(dev):
        check(getattr(lib(), name)(*args, stream_ptr(dev)), name)


# ------------------------------------------------------------------------------------------------
# tensor-level helpers (op level; the model-level fast path lives in engine.py)
# ------------------------------------------------------------------------------------------------
def split(x: torch.Tensor, relu: bool = False, out=None):
    """fp32 [..., C] contiguous -> (hi, lo) bf16 planes of the same shape (`out`: existing planes to overwrite)."""
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    c = x.shape[-1]
    rows = x.numel() // c
    if out is not None:
        hi, lo = out
        assert hi.numel() == x.numel() and lo.numel() == x.numel() and hi.dtype == torch.bfloat16 and hi.device == x.device
    else:
        hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        lo = torch.empty_like(hi)
    call("s3r_split", x, ptr(x), c, ptr(hi), ptr(lo), c, 0, rows, c, int(relu))
    return hi, lo


def layernorm(x, w, b, eps, want_f32=True, want_planes=False):
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    c = x.shape[-1]
    rows = x.numel() // c
    out = torch.empty_like(x) if want_f32 else None
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if want_planes else None
    lo = torch.empty_like(hi) if want_planes else None
    call("s3r_layernorm", x, ptr(x), c, ptr(w), ptr(b), 0, 0, float(eps), rows, c, ptr(out), c, ptr(hi), ptr(lo), c, 0, 0)
    return out, hi, lo


def gemm(desc: GemmDesc, device=None):
    """device: the device the descriptor's pointers live on (default: the current device)."""
    call("s3r_gemm", device, C.byref(desc))


def linear(x_planes, w_planes, bias=None, act=ACT_NONE, res=None, want_f32=True, want_planes=False, plane_relu=False,
           groups=1, force_bn=0):
    """y = act(x @ W^T + bias) + res.  x planes [G*rows, K], W planes [G*N, K]."""
    xh, xl = x_planes
    wh, wl = w_planes
    K = xh.shape[-1]
    rows = xh.numel() // K // groups
    N = wh.shape[0] // groups
    dev = xh.device
    out = torch.empty((groups * rows, N), dtype=torch.float32, device=dev) if want_f32 else None
    oh = torch.empty((groups * rows, N), dtype=torch.bfloat16, device=dev) if want_planes else None
    ol = torch.empty_like(oh) if want_planes else None
    d = GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, 1, 1, rows, K, 1, N
    d.epi, d.act, d.plane_relu, d.force_bn = EPI_PLAIN, act, int(plane_relu), force_bn
    d.bias = bias.data_ptr() if bias is not None else None
    if res is not None:
        d.res1, d.ldr1 = res.data_ptr(), N
    if out is not None:
        d.out_f32, d.ldo = out.data_ptr(), N
    if oh is not None:
        d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), N
    gemm(d, dev)
    return out, oh, ol


def conv_wgrad(dy_planes, x_planes, taps: int) -> torch.Tensor:
    """Conv weight gradient over pixels: dy planes [nb, h, w, n], x planes [nb, h, w, kc] (NHWC, contiguous) ->
    fp32 dW [n, taps, kc] (taps 9: the 3x3 stride-1 pad-1 shifts).  Bitwise reproducible."""
    yh, yl = dy_planes
    xh, xl = x_planes
    nb, h, w, n = yh.shape
    kc = xh.shape[-1]
    assert tuple(xh.shape[:3]) == (nb, h, w) and yh.is_contiguous() and xh.is_contiguous(), (tuple(yh.shape), tuple(xh.shape))
    ws_bytes = lib().s3r_conv_wgrad_workspace_bytes(nb, h, w, n, kc, taps)
    if ws_bytes == 0:
        raise S3RError(f"s3r_conv_wgrad: unsupported shape nb={nb} h={h} w={w} n={n} kc={kc} taps={taps}")
    dev = yh.device
    ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=dev)
    dw = torch.empty((n, taps, kc), dtype=torch.float32, device=dev)
    call("s3r_conv_wgrad", dev, ptr(yh), ptr(yl), n, ptr(xh), ptr(xl), kc, nb, h, w, n, kc, taps, ptr(ws), ws_bytes, ptr(dw))
    return dw


def col2im_3x3s2(cols: torch.Tensor, nb: int, h: int, w: int, c: int) -> torch.Tensor:
    """Adjoint of s3r_im2col_3x3s2: fp32 cols [nb*ho*wo, 9*c] -> fp32 [nb, h, w, c]."""
    assert cols.dtype == torch.float32 and cols.is_cuda and cols.is_contiguous()
    out = torch.empty((nb, h, w, c), dtype=torch.float32, device=cols.device)
    call("s3r_col2im_3x3s2", cols, ptr(cols), nb, h, w, c, (h + 1) // 2, (w + 1) // 2, ptr(out))
    return out


def conf_score(conf: torch.Tensor) -> torch.Tensor:
    """mean((conf-1)/conf) over all elements, as a 1-element device tensor."""
    assert conf.is_cuda and conf.dtype == torch.float32 and conf.is_contiguous()
    scratch = torch.empty(256, dtype=torch.float32, device=conf.device)
    out = torch.empty(1, dtype=torch.float32, device=conf.device)
    call("s3r_conf_score", conf, ptr(conf), conf.numel(), ptr(scratch), ptr(out))
    return out


def conf_score_batched(conf: torch.Tensor) -> torch.Tensor:
    """conf [2, B, H, W] (the engine's heads output) -> [2, B]: `conf_score` of every image, bitwise, in one launch pair."""
    assert conf.is_cuda and conf.dtype == torch.float32 and conf.is_contiguous() and conf.dim() == 4 and conf.shape[0] == 2
    B, hw = conf.shape[1], conf.shape[2] * conf.shape[3]
    scratch = torch.empty(2 * B * 256, dtype=torch.float32, device=conf.device)
    out = torch.empty(2, B, dtype=torch.float32, device=conf.device)
    call("s3r_conf_score_batched", conf, ptr(conf), B, hw, ptr(scratch), ptr(out))
    return out


def dropout_mask(shape, seed: int, p: float, device) -> torch.Tensor:
    """Keep-scale (0 or 1 / (1 - p)) of every element of a [..., len] attention tensor under the Philox mask the
    training-mode memory read applies for `seed` (s3r_engine_memory_read_train); flat index = row-major position."""
    out = torch.empty(shape, dtype=torch.float32, device=device)
    call("s3r_dropout_mask", out, ptr(out), out.numel(), int(seed) & 0xFFFFFFFFFFFFFFFF, float(p))
    return out
