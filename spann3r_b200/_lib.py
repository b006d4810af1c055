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
    ]


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
    "s3r_gemm": (_i, [C.POINTER(GemmDesc), _vp]),
    "s3r_gemm_tile_n": (_i, [C.POINTER(GemmDesc)]),
    "s3r_attention": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i64, _vp]),
    "s3r_conf_score": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "s3r_dropout_mask": (_i, [_vp, _i64, C.c_uint64, _f, _vp]),
    "s3r_set_option": (_i, [C.c_char_p, _i]),
    "s3r_focal_weiszfeld": (_i, [_vp, _i, _i, _i, _f, _f, _i, _f, _f, _vp, _vp, _vp]),
    "s3r_focal_median": (_i, [_vp, _i, _i, _i, _f, _f, _f, _f, _vp, _vp, _vp]),
    "s3r_pnp_workspace_bytes": (C.c_size_t, [_i, _i]),
    "s3r_pnp_ransac": (_i, [_vp, _vp, _i, _i64, _i, C.c_double, C.c_double, C.c_double, C.c_double, _f, _i, _i, C.c_uint64,
                            _vp, _vp, _vp, _vp]),
    "s3r_resample_h_u8": (_i, [_vp, _i64, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "s3r_resample_v_u8_norm": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp, _vp]),
}

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
        _ENGINE_PROTOS_HOOK(L)
        _lib = L
    return _lib


def _ENGINE_PROTOS_HOOK(L):  # replaced by engine.py when it defines more entry points
    for name, (res, args) in _EXTRA_PROTOS.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args


_EXTRA_PROTOS: dict = {}


def register_protos(protos: dict):
    _EXTRA_PROTOS.update(protos)
    if _lib is not None:
        _ENGINE_PROTOS_HOOK(_lib)


def declared_symbols():
    return list(_PROTOS) + list(_EXTRA_PROTOS)


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
    with on_device(x):
        check(lib().s3r_split(ptr(x), c, ptr(hi), ptr(lo), c, 0, rows, c, int(relu), stream_ptr(x.device)), "s3r_split")
    return hi, lo


def layernorm(x, w, b, eps, want_f32=True, want_planes=False):
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    c = x.shape[-1]
    rows = x.numel() // c
    out = torch.empty_like(x) if want_f32 else None
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if want_planes else None
    lo = torch.empty_like(hi) if want_planes else None
    with on_device(x):
        check(lib().s3r_layernorm(ptr(x), c, ptr(w), ptr(b), 0, 0, float(eps), rows, c, ptr(out), c, ptr(hi), ptr(lo), c, 0,
                                  0, stream_ptr(x.device)), "s3r_layernorm")
    return out, hi, lo


def gemm(desc: GemmDesc, device=None):
    """device: the device the descriptor's pointers live on (default: the current device)."""
    if device is None:
        return check(lib().s3r_gemm(C.byref(desc), stream_ptr()), "s3r_gemm")
    with on_device(device):
        check(lib().s3r_gemm(C.byref(desc), stream_ptr(device)), "s3r_gemm")


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


def conf_score(conf: torch.Tensor) -> torch.Tensor:
    """mean((conf-1)/conf) over all elements, as a 1-element device tensor."""
    assert conf.is_cuda and conf.dtype == torch.float32 and conf.is_contiguous()
    scratch = torch.empty(256, dtype=torch.float32, device=conf.device)
    out = torch.empty(1, dtype=torch.float32, device=conf.device)
    with on_device(conf):
        check(lib().s3r_conf_score(ptr(conf), conf.numel(), ptr(scratch), ptr(out), stream_ptr(conf.device)), "s3r_conf_score")
    return out


def dropout_mask(shape, seed: int, p: float, device) -> torch.Tensor:
    """Keep-scale (0 or 1 / (1 - p)) of every element of a [..., len] attention tensor under the Philox mask the
    training-mode memory read applies for `seed` (s3r_engine_memory_read_train); flat index = row-major position."""
    out = torch.empty(shape, dtype=torch.float32, device=device)
    with on_device(out):
        check(lib().s3r_dropout_mask(ptr(out), out.numel(), int(seed) & 0xFFFFFFFFFFFFFFFF, float(p), stream_ptr(out.device)),
              "s3r_dropout_mask")
    return out
