"""ctypes binding of libdvla_sm90.so (include/dvla.h).  This is the only place Python touches the C ABI.

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
PyTorch is used for device memory and streams only (tensor.data_ptr(), torch.cuda.current_stream()).
"""
from __future__ import annotations

import ctypes as C
import threading
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdvla_sm90.so")

ACT_NONE, ACT_GELU_ERF, ACT_GELU_TANH, ACT_QUICK_GELU, ACT_RELU, ACT_SILU = range(6)
ACT_IDS = {None: 0, "none": 0, "gelu": 1, "gelu_erf": 1, "gelu_tanh": 2, "gelu_new": 2, "quick_gelu": 3, "relu": 4,
           "silu": 5}

_vp, _i64, _i32, _f32, _u64 = C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_uint64


class GemmArgs(C.Structure):
    _fields_ = [("a", _vp), ("b", _vp), ("out", _vp), ("bias", _vp), ("residual", _vp), ("aux_out", _vp),
                ("aux_in", _vp), ("M", _i64), ("N", _i64), ("K", _i64), ("lda", _i64), ("ldb", _i64), ("ldo", _i64),
                ("ldr", _i64), ("ld_aux", _i64), ("a_mn_major", _i32), ("b_mn_major", _i32), ("act", _i32),
                ("out_fp32", _i32), ("alpha", _f32), ("dropout_p", _f32), ("dropout_seed", _u64), ("dropout_seed_ptr", _vp),
                ("workspace", _vp), ("workspace_bytes", _i64)]


class GemmPlanInfo(C.Structure):
    _fields_ = [(n, _i32) for n in ("kernel", "tile_m", "tile_n", "m_tiles", "n_tiles", "k_blocks", "k_splits", "kb_per_split",
                                    "atomic_out", "tail_first", "tail_splits", "tail_kbps", "units", "grid_ctas")]


class LayerNormFwdArgs(C.Structure):
    _fields_ = [("x", _vp), ("gamma", _vp), ("beta", _vp), ("y", _vp), ("mean", _vp), ("rstd", _vp), ("rows", _i64),
                ("D", _i64), ("ldx", _i64), ("ldy", _i64), ("eps", _f32)]


class LayerNormBwdArgs(C.Structure):
    _fields_ = [("dy", _vp), ("x", _vp), ("gamma", _vp), ("mean", _vp), ("rstd", _vp), ("dx", _vp), ("dgamma", _vp),
                ("dbeta", _vp), ("rows", _i64), ("D", _i64), ("ld", _i64), ("dres", _vp)]


class AttnFwdArgs(C.Structure):
    _fields_ = [("q", _vp), ("k", _vp), ("v", _vp), ("o", _vp), ("lse", _vp), ("mask", _vp), ("tile_flags", _vp),
                ("B", _i64), ("H", _i64), ("Lq", _i64), ("Lk", _i64),
                ("q_sb", _i64), ("q_ss", _i64), ("q_sh", _i64), ("k_sb", _i64), ("k_ss", _i64), ("k_sh", _i64),
                ("v_sb", _i64), ("v_ss", _i64), ("v_sh", _i64), ("o_sb", _i64), ("o_ss", _i64), ("o_sh", _i64),
                ("mask_words", _i32), ("scale", _f32), ("dropout_p", _f32), ("dropout_seed", _u64), ("dropout_seed_ptr", _vp),
                ("key_bias", _vp), ("head_dim", _i64), ("mask_index", _vp), ("mask_stride", _i64), ("flags_stride", _i64)]


class AttnBwdArgs(C.Structure):
    _fields_ = [("q", _vp), ("k", _vp), ("v", _vp), ("o", _vp), ("d_o", _vp), ("lse", _vp), ("delta", _vp),
                ("dq", _vp), ("dk", _vp), ("dv", _vp), ("mask", _vp), ("tile_flags", _vp),
                ("B", _i64), ("H", _i64), ("Lq", _i64), ("Lk", _i64),
                ("q_sb", _i64), ("q_ss", _i64), ("q_sh", _i64), ("k_sb", _i64), ("k_ss", _i64), ("k_sh", _i64),
                ("v_sb", _i64), ("v_ss", _i64), ("v_sh", _i64), ("o_sb", _i64), ("o_ss", _i64), ("o_sh", _i64),
                ("do_sb", _i64), ("do_ss", _i64), ("do_sh", _i64),
                ("dq_sb", _i64), ("dq_ss", _i64), ("dq_sh", _i64), ("dk_sb", _i64), ("dk_ss", _i64), ("dk_sh", _i64),
                ("dv_sb", _i64), ("dv_ss", _i64), ("dv_sh", _i64),
                ("mask_words", _i32), ("scale", _f32), ("dropout_p", _f32), ("dropout_seed", _u64), ("dropout_seed_ptr", _vp),
                ("mask_t", _vp), ("mask_t_words", _i32), ("key_bias", _vp), ("head_dim", _i64)]


class AdamWArgs(C.Structure):
    _fields_ = [("p", _vp), ("g", _vp), ("m", _vp), ("v", _vp), ("n", _i64), ("sumsq", _vp), ("lr", _vp),
                ("step", _vp), ("beta1", _f32), ("beta2", _f32), ("eps", _f32), ("weight_decay", _f32),
                ("max_norm", _f32), ("grad_scale", _f32), ("zero_grad", _i32)]


class AdamWMasterArgs(C.Structure):
    _fields_ = [("p32", _vp), ("p", _vp), ("g", _vp), ("m", _vp), ("v", _vp), ("n", _i64), ("sumsq", _vp), ("lr", _vp),
                ("step", _vp), ("beta1", _f32), ("beta2", _f32), ("eps", _f32), ("weight_decay", _f32),
                ("max_norm", _f32), ("grad_scale", _f32), ("zero_grad", _i32)]


class ImageFnArgs(C.Structure):
    _fields_ = [("frames", _vp), ("out", _vp), ("n", _i64), ("h", _i64), ("w", _i64), ("c", _i64), ("xbounds", _vp),
                ("xcoeffs", _vp), ("ybounds", _vp), ("ycoeffs", _vp), ("lut", _vp), ("flip_vertical", _i32), ("out_dtype", _i32)]


class DitBlockWeights(C.Structure):
    _fields_ = [(n, _vp) for n in ("qkv_w", "qkv_b", "proj_w", "proj_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b")]


class DitSamplerArgs(C.Structure):
    _fields_ = [("blocks", C.POINTER(DitBlockWeights))] + \
               [(n, _i64) for n in ("depth", "hidden", "heads", "mlp", "token", "freq", "channels", "T", "batch")] + \
               [(n, _vp) for n in ("x_w", "x_b", "t0_w", "t0_b", "t2_w", "t2_b", "z_w", "z_b", "uncondition", "pos", "final_w",
                                   "final_b", "z", "noise", "out")] + \
               [("timestep_map", C.POINTER(_i32)), ("sqrt_recip_alphas_cumprod", C.POINTER(_f32)),
                ("sqrt_recipm1_alphas_cumprod", C.POINTER(_f32)), ("alphas_cumprod_prev", C.POINTER(_f32)),
                ("n_steps", _i64), ("cfg_scale", _f32), ("workspace", _vp), ("workspace_bytes", _i64),
                ("integrator", _i64), ("t_values", C.POINTER(_f32))]


DIT_DDIM, DIT_FM_EULER = 0, 1     # dvla_dit_sampler_args.integrator


# name -> (restype, argtypes) of every function include/dvla.h declares; tests/test_abi_cpu.py checks it against the header.
# Pointers (device buffers, args structs, streams) are c_void_p: it takes tensor.data_ptr(), None and C.byref(...).
_int = C.c_int
PROTOTYPES = {
    "dvla_version": (_int, []),
    "dvla_last_error": (C.c_char_p, []),
    "dvla_launch_count": (_i64, []),
    "dvla_gemm": (_int, [_vp, _vp]),
    "dvla_gemm_plan": (_int, [_vp, _vp]),
    "dvla_gemm_plan_unit": (_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "dvla_layernorm_fwd": (_int, [_vp, _vp]),
    "dvla_layernorm_bwd": (_int, [_vp, _vp]),
    "dvla_attn_fwd": (_int, [_vp, _vp]),
    "dvla_attn_bwd": (_int, [_vp, _vp]),
    "dvla_attn_mask_tiles": (_int, [_vp, _i32, _i64, _i64, _vp, _vp]),
    "dvla_attn_mask_obs_drop": (_int, [_vp, _vp, _vp, _i32, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _u64, _vp, _vp]),
    "dvla_colsum_accum": (_int, [_vp, _i64, _i64, _i64, _vp, _vp]),
    "dvla_accum_fp32_into_bf16": (_int, [_vp, _vp, _i64, _vp]),
    "dvla_dropout": (_int, [_vp, _vp, _i64, _i64, _i64, _i64, _f32, _u64, _vp, _vp]),
    "dvla_cat_broadcast": (_int, [_vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp]),
    "dvla_act_bwd": (_int, [_vp, _vp, _vp, _i64, _i32, _vp]),
    "dvla_act_bwd_colsum": (_int, [_vp, _vp, _vp, _i64, _i64, _i32, _vp, _vp]),
    "dvla_mse_loss": (_int, [_vp, _vp, _vp, _i64, _i64, _f32, _vp, _vp, _vp]),
    "dvla_cosine_loss": (_int, [_vp, _vp, _i64, _i64, _f32, _vp, _vp, _vp]),
    "dvla_silog_stats": (_int, [_vp, _vp, _i64, _vp, _vp]),
    "dvla_silog_finish": (_int, [_vp, _vp, _i64, _vp, _f32, _f32, _vp, _vp, _vp]),
    "dvla_sumsq": (_int, [_vp, _i64, _vp, _vp]),
    "dvla_adamw": (_int, [_vp, _vp]),
    "dvla_adamw_master": (_int, [_vp, _vp]),
    "dvla_grad_clip_scale": (_int, [_vp, _i64, _vp, _f32, _f32, _vp]),
    "dvla_dit_sampler_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64, _i64]),
    "dvla_dit_ddim_sample": (_int, [_vp, _vp]),
    "dvla_shift_crop": (_int, [_vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _vp]),
    "dvla_resize_nearest": (_int, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _i32, _vp]),
    "dvla_image_fn": (_int, [_vp, _vp]),
    "dvla_bicubic_taps": (_i32, [_i64, _i64]),
    "dvla_bicubic_coeffs": (_int, [_i64, _i64, _i64, _i64, _vp, _vp]),
    "dvla_set_sm_budget": (_int, [_int]),
    "dvla_attn_bwd_workspace_bytes": (_i64, [_i64, _i64, _i64]),
    "dvla_silog_workspace_bytes": (_i64, []),
    "dvla_gemm_workspace_bytes": (_i64, [_vp]),
}
EXPORTS = sorted(PROTOTYPES)

_lib = None


def load() -> C.CDLL:
    """Load the shared library; raises if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m dreamvla_b200.build` (nvcc, sm_90a). "
            "dreamvla_b200 has no CPU or PyTorch fallback for its kernels.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        if not hasattr(lib, name):
            raise RuntimeError(f"{LIB_PATH} does not export {name} (stale build? run `python -m dreamvla_b200.build`)")
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def launch_count() -> int:
    return int(load().dvla_launch_count())


def _call(name: str, *args) -> int:
    """Calls library function `name` and returns its result; a negative dvla_status raises RuntimeError with the text of
    dvla_last_error()."""
    rc = getattr(load(), name)(*args)
    if rc < 0:
        raise RuntimeError(f"{name} failed ({rc}): {load().dvla_last_error().decode()}")
    return rc


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def _need_cuda(*ts) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("dreamvla_b200 kernels need CUDA tensors (no CPU fallback)")


# ----------------------------------------------------------------------------------------------------------------------
# raw op wrappers (no autograd)
# ----------------------------------------------------------------------------------------------------------------------
_gemm_ws = {}
_gemm_ws_lock = threading.Lock()


def gemm_workspace(device):
    """The GEMM scratch (fp32 partial tiles + arrival counters, include/dvla.h `dvla_gemm_args.workspace`) of the CURRENT
    stream of `device`: one zero-initialised buffer per (device, stream), kept for the life of the process -- the kernels
    leave its counter block zero again, and calls on one stream are ordered, so they can share it."""
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    ws = _gemm_ws.get(key)
    if ws is None:
        with _gemm_ws_lock:                 # forward thread and autograd's backward thread may both arrive here first
            ws = _gemm_ws.get(key)
            if ws is None:
                ws = _gemm_ws[key] = torch.zeros(int(load().dvla_gemm_workspace_bytes(None)), device=device, dtype=torch.uint8)
    return ws


def gemm(a, b, **kw):
    """out[M,N] = epi(alpha * A @ B^T).  a: [M,K] (or [K,M] if a_mn), b: [N,K] (or [K,N] if b_mn); 2-D, unit inner stride.
    Keywords: see _gemm_args."""
    args, out = _gemm_args(a, b, **kw)
    _call("dvla_gemm", C.byref(args), _stream())
    return out


def gemm_plan(a, b, **kw) -> GemmPlanInfo:
    """What gemm(a, b, **kw) would launch on the current device (dvla_gemm_plan of the same arguments); launches nothing."""
    args, _ = _gemm_args(a, b, **kw)
    info = GemmPlanInfo()
    _call("dvla_gemm_plan", C.byref(args), C.byref(info))
    return info


def _gemm_args(a, b, *, a_mn=False, b_mn=False, bias=None, act=0, residual=None, aux_out=None, aux_in=None, out=None,
               out_dtype=torch.bfloat16, alpha=1.0, dropout_p=0.0, dropout_seed=0, dropout_seed_ptr=None):
    _need_cuda(a, b)
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1, (a.shape, a.stride(), b.shape, b.stride())
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=out_dtype)
    assert out.shape == (M, N) and out.stride(1) == 1
    args = GemmArgs()
    args.a, args.b, args.out = a.data_ptr(), b.data_ptr(), out.data_ptr()
    args.bias = _ptr(bias)
    if residual is not None:
        assert residual.shape == (M, N) and residual.stride(1) == 1 and residual.dtype == out.dtype
        args.residual, args.ldr = residual.data_ptr(), residual.stride(0)
    if aux_out is not None:
        assert aux_out.shape == (M, N) and aux_out.stride(1) == 1 and aux_out.dtype == torch.bfloat16
        args.aux_out, args.ld_aux = aux_out.data_ptr(), aux_out.stride(0)
    if aux_in is not None:
        assert aux_in.shape == (M, N) and aux_in.stride(1) == 1 and aux_in.dtype == torch.bfloat16
        args.aux_in, args.ld_aux = aux_in.data_ptr(), aux_in.stride(0)
    args.M, args.N, args.K = M, N, K
    args.lda, args.ldb, args.ldo = a.stride(0), b.stride(0), out.stride(0)
    args.a_mn_major, args.b_mn_major = int(a_mn), int(b_mn)
    args.act = int(act)
    args.out_fp32 = int(out.dtype == torch.float32)
    args.alpha = float(alpha)
    args.dropout_p = float(dropout_p)
    args.dropout_seed = int(dropout_seed)
    args.dropout_seed_ptr = _ptr(dropout_seed_ptr)
    ws = gemm_workspace(a.device)
    args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
    return args, out


def layernorm_fwd(x2d, gamma, beta, eps, save_stats=True):
    _need_cuda(x2d)
    rows, D = x2d.shape
    assert x2d.stride(1) == 1 and x2d.dtype == torch.bfloat16
    y = torch.empty((rows, D), device=x2d.device, dtype=torch.bfloat16)
    mean = torch.empty(rows, device=x2d.device, dtype=torch.float32) if save_stats else None
    rstd = torch.empty(rows, device=x2d.device, dtype=torch.float32) if save_stats else None
    a = LayerNormFwdArgs(x2d.data_ptr(), _ptr(gamma), _ptr(beta), y.data_ptr(), _ptr(mean), _ptr(rstd), rows, D,
                         x2d.stride(0), y.stride(0), float(eps))
    _call("dvla_layernorm_fwd", C.byref(a), _stream())
    return y, mean, rstd


def layernorm_bwd(dy2d, x2d, gamma, mean, rstd, dgamma_f32, dbeta_f32, dres2d=None):
    """dx = LN'(dy) [+ dres2d]; dres2d = gradient arriving at x through a residual branch (same shape as x2d)."""
    rows, D = x2d.shape
    assert dy2d.is_contiguous() and x2d.is_contiguous()
    assert dres2d is None or (dres2d.is_contiguous() and dres2d.shape == x2d.shape and dres2d.dtype == torch.bfloat16)
    dx = torch.empty_like(x2d)
    a = LayerNormBwdArgs(dy2d.data_ptr(), x2d.data_ptr(), _ptr(gamma), mean.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
                         _ptr(dgamma_f32), _ptr(dbeta_f32), rows, D, D, _ptr(dres2d))
    _call("dvla_layernorm_bwd", C.byref(a), _stream())
    return dx


def _bsh(t, hd=64):
    """[B, L, H, hd] view -> (batch, seq, head) element strides."""
    assert t.dim() == 4 and t.shape[-1] == hd and t.stride(3) == 1 and t.dtype == torch.bfloat16, (t.shape, t.stride())
    return t.stride(0), t.stride(1), t.stride(2)


def attn_fwd(q, k, v, scale, mask_bits=None, tile_flags=None, dropout_p=0.0, dropout_seed=0, need_lse=True,
             dropout_seed_ptr=None, key_bias=None, mask_index=None):
    """q [B,Lq,H,hd], k/v [B,Lk,H,hd] (arbitrary batch/seq/head strides) -> o [B,Lq,H,hd] contiguous, lse [B,H,Lq].
    hd = 64, or 96 where the short-sequence kernels run (the library refuses other cases).
    mask_index: device int32 [B] selecting, per batch, one matrix of the stacks mask_bits [n, Lq, words] / tile_flags
    [n, nqt, nkt] (contiguous)."""
    _need_cuda(q, k, v)
    B, Lq, H, hd = q.shape
    Lk = k.shape[1]
    o = torch.empty((B, Lq, H, hd), device=q.device, dtype=torch.bfloat16)
    lse = torch.empty((B, H, Lq), device=q.device, dtype=torch.float32) if need_lse else None
    a = AttnFwdArgs()
    a.q, a.k, a.v, a.o, a.lse = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), _ptr(lse)
    a.mask, a.tile_flags = _ptr(mask_bits), _ptr(tile_flags)
    a.B, a.H, a.Lq, a.Lk, a.head_dim = B, H, Lq, Lk, hd
    a.q_sb, a.q_ss, a.q_sh = _bsh(q, hd)
    a.k_sb, a.k_ss, a.k_sh = _bsh(k, hd)
    a.v_sb, a.v_ss, a.v_sh = _bsh(v, hd)
    a.o_sb, a.o_ss, a.o_sh = _bsh(o, hd)
    a.mask_words = 0 if mask_bits is None else mask_bits.shape[-1]
    a.scale, a.dropout_p, a.dropout_seed = float(scale), float(dropout_p), int(dropout_seed)
    a.dropout_seed_ptr = _ptr(dropout_seed_ptr)
    if mask_index is not None:
        assert mask_index.dtype == torch.int32 and mask_index.is_contiguous() and mask_index.numel() == B
        assert mask_bits.dim() == 3 and mask_bits.is_contiguous() and tile_flags.dim() == 3 and tile_flags.is_contiguous()
        a.mask_index, a.mask_stride, a.flags_stride = mask_index.data_ptr(), mask_bits[0].numel(), tile_flags[0].numel()
    if key_bias is not None:
        assert key_bias.dtype == torch.float32 and key_bias.is_contiguous() and key_bias.numel() == Lk
        a.key_bias = key_bias.data_ptr()
    _call("dvla_attn_fwd", C.byref(a), _stream())
    return o, lse


def attn_bwd(q, k, v, o, d_o, lse, scale, dq, dk, dv, mask_bits=None, tile_flags=None, dropout_p=0.0, dropout_seed=0,
             dropout_seed_ptr=None, key_bias=None):
    B, Lq, H, hd = q.shape
    Lk = k.shape[1]
    ws = load().dvla_attn_bwd_workspace_bytes(B, H, Lq)
    delta = torch.empty(ws // 4, device=q.device, dtype=torch.float32)
    a = AttnBwdArgs()
    a.q, a.k, a.v, a.o, a.d_o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr()
    a.lse, a.delta = lse.data_ptr(), delta.data_ptr()
    a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    a.mask, a.tile_flags = _ptr(mask_bits), _ptr(tile_flags)
    a.B, a.H, a.Lq, a.Lk, a.head_dim = B, H, Lq, Lk, hd
    a.q_sb, a.q_ss, a.q_sh = _bsh(q, hd)
    a.k_sb, a.k_ss, a.k_sh = _bsh(k, hd)
    a.v_sb, a.v_ss, a.v_sh = _bsh(v, hd)
    a.o_sb, a.o_ss, a.o_sh = _bsh(o, hd)
    a.do_sb, a.do_ss, a.do_sh = _bsh(d_o, hd)
    a.dq_sb, a.dq_ss, a.dq_sh = _bsh(dq, hd)
    a.dk_sb, a.dk_ss, a.dk_sh = _bsh(dk, hd)
    a.dv_sb, a.dv_ss, a.dv_sh = _bsh(dv, hd)
    a.mask_words = 0 if mask_bits is None else mask_bits.shape[1]
    a.scale, a.dropout_p, a.dropout_seed = float(scale), float(dropout_p), int(dropout_seed)
    a.dropout_seed_ptr = _ptr(dropout_seed_ptr)
    a.key_bias = _ptr(key_bias)
    _call("dvla_attn_bwd", C.byref(a), _stream())


def attn_mask_tiles(mask_bits, Lq, Lk, out=None):
    """Tile flags [ceil(Lq/64), ceil(Lk/64)] uint8 of a bit mask; `out` refreshes an existing flags buffer in place."""
    nqt, nkt = (Lq + 63) // 64, (Lk + 63) // 64
    flags = torch.empty((nqt, nkt), device=mask_bits.device, dtype=torch.uint8) if out is None else out
    assert flags.shape == (nqt, nkt) and flags.dtype == torch.uint8 and flags.is_contiguous()
    _call("dvla_attn_mask_tiles", mask_bits.data_ptr(), mask_bits.shape[1], Lq, Lk, flags.data_ptr(), _stream())
    return flags


def attn_mask_obs_drop(base_bits, bits, flags, K, n_tok, num_A, n_obs, n_act, count, seed, seed_ptr=None):
    """bits = base_bits with `count` observation columns per timestep hidden from that timestep's action rows, flags = its
    tile flags (include/dvla.h dvla_attn_mask_obs_drop); both written in place, capturable in a CUDA graph."""
    _need_cuda(base_bits, bits, flags, seed_ptr)
    L_, W = base_bits.shape
    assert bits.shape == (L_, W) and base_bits.dtype == bits.dtype == torch.int32
    assert base_bits.is_contiguous() and bits.is_contiguous() and flags.is_contiguous() and flags.dtype == torch.uint8
    assert flags.shape == ((L_ + 63) // 64, (L_ + 63) // 64)
    assert seed_ptr is None or (seed_ptr.dtype == torch.int64 and seed_ptr.numel() >= 1)
    _call("dvla_attn_mask_obs_drop", base_bits.data_ptr(), bits.data_ptr(), flags.data_ptr(), W, L_, K, n_tok, num_A, n_obs,
          n_act, count, int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(seed_ptr), _stream())


def colsum_accum(x2d, out_f32):
    rows, N = x2d.shape
    assert x2d.stride(1) == 1
    _call("dvla_colsum_accum", x2d.data_ptr(), rows, N, x2d.stride(0), out_f32.data_ptr(), _stream())


def accum_fp32_into_bf16(src_f32, dst_bf16):
    assert src_f32.is_contiguous() and dst_bf16.is_contiguous() and src_f32.numel() == dst_bf16.numel()
    _call("dvla_accum_fp32_into_bf16", src_f32.data_ptr(), dst_bf16.data_ptr(), src_f32.numel(), _stream())


def dropout(x2d, p, seed, out=None, seed_ptr=None):
    rows, N = x2d.shape
    assert x2d.stride(1) == 1
    y = torch.empty((rows, N), device=x2d.device, dtype=torch.bfloat16) if out is None else out
    _call("dvla_dropout", x2d.data_ptr(), y.data_ptr(), rows, N, x2d.stride(0), y.stride(0), p, seed, _ptr(seed_ptr),
          _stream())
    return y


_DT = {torch.float32: 0, torch.bfloat16: 1}


def shift_crop(x, shifts_xy, pad, out_dtype=None):
    """out[i, c, y, x] = x[i, c, clamp(y + sy_i - pad), clamp(x + sx_i - pad)]: RandomShiftsAug for given shifts (include/dvla.h).
    x [n, c, H, W] fp32 / bf16 contiguous, shifts_xy int32 [n, 2] on the same device."""
    _need_cuda(x, shifts_xy)
    assert x.dim() == 4 and x.is_contiguous() and x.dtype in _DT
    n, c, h, w = x.shape
    assert shifts_xy.dtype == torch.int32 and shifts_xy.shape == (n, 2) and shifts_xy.is_contiguous()
    out = torch.empty_like(x, dtype=out_dtype or x.dtype)
    _call("dvla_shift_crop", x.data_ptr(), out.data_ptr(), shifts_xy.data_ptr(), n, c, h, w, int(pad), _DT[x.dtype],
          _DT[out.dtype], _stream())
    return out


def resize_nearest(x, hout, wout, out_dtype=torch.float32):
    """torchvision Resize((hout, wout), NEAREST) of a float32 [..., Hin, Win] tensor (depth_image_fn, include/dvla.h)."""
    _need_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() >= 2
    hin, win = x.shape[-2:]
    n = x.numel() // (hin * win)
    out = torch.empty((*x.shape[:-2], hout, wout), device=x.device, dtype=out_dtype)
    _call("dvla_resize_nearest", x.data_ptr(), out.data_ptr(), n, hin, win, hout, wout, _DT[out_dtype], _stream())
    return out


IMAGE_FN_SIZE = 224


def image_fn_geometry(h, w, size=IMAGE_FN_SIZE):
    """torchvision `Resize(size)` (short side -> size, long side int(size * long / short)) + `CenterCrop(size)` of an h x w
    frame -> (resized h, resized w, crop top, crop left); include/dvla.h dvla_image_fn."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    rh, rw = (new_long, size) if w <= h else (size, new_long)
    return rh, rw, int(round((rh - size) / 2.0)), int(round((rw - size) / 2.0))


def bicubic_coeffs(in_size, out_size, first, count):
    """Pillow's bicubic bounds / int32 coefficients of outputs [first, first + count) of a line resized from in_size to
    out_size (host only, no GPU): (bounds int32 [count, 2] = (first input pixel, taps used), coeffs int32 [count, taps])."""
    taps = _call("dvla_bicubic_taps", in_size, out_size)
    bounds = torch.zeros((count, 2), dtype=torch.int32)
    coeffs = torch.zeros((count, taps), dtype=torch.int32)
    _call("dvla_bicubic_coeffs", in_size, out_size, first, count, bounds.data_ptr(), coeffs.data_ptr())
    return bounds, coeffs


_image_fn_tables = {}


def image_fn_tables(h, w, device):
    """Device copies of the coefficient tables of an h x w frame ((xbounds, xcoeffs, ybounds, ycoeffs)), built once per
    (device, h, w).  The first call for a frame size uploads them: make it outside CUDA-graph capture."""
    key = (device.index if device.index is not None else torch.cuda.current_device(), int(h), int(w))
    t = _image_fn_tables.get(key)
    if t is None:
        rh, rw, top, left = image_fn_geometry(h, w)
        xb, xc = bicubic_coeffs(w, rw, left, IMAGE_FN_SIZE)
        yb, yc = bicubic_coeffs(h, rh, top, IMAGE_FN_SIZE)
        t = _image_fn_tables[key] = tuple(v.to(device) for v in (xb, xc, yb, yc))
    return t


def image_fn(frames, lut, out_dtype=torch.float32, flip_vertical=False):
    """CLIP `_transform(224)` of uint8 frames [n, h, w, 3] (contiguous, HWC) -> [n, 3, 224, 224] `out_dtype` (fp32 / bf16):
    Pillow-exact bicubic resize of the short side to 224, centre crop, then out = lut[c, value] with lut fp32 [3, 256]
    (include/dvla.h dvla_image_fn).  flip_vertical reads every frame bottom-up."""
    _need_cuda(frames, lut)
    assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.is_contiguous(), (frames.dtype, frames.shape)
    assert lut.dtype == torch.float32 and lut.shape == (3, 256) and lut.is_contiguous()
    n, h, w, c = frames.shape
    out = torch.empty((n, 3, IMAGE_FN_SIZE, IMAGE_FN_SIZE), device=frames.device, dtype=out_dtype)
    if n == 0:
        return out
    xb, xc, yb, yc = image_fn_tables(h, w, frames.device)
    a = ImageFnArgs(frames.data_ptr(), out.data_ptr(), n, h, w, c, xb.data_ptr(), xc.data_ptr(), yb.data_ptr(), yc.data_ptr(),
                    lut.data_ptr(), int(bool(flip_vertical)), _DT[out_dtype])
    _call("dvla_image_fn", C.byref(a), _stream())
    return out


def act_bwd(dy, pre, act, colsum_out=None):
    """dx = dy * act'(pre); with `colsum_out` (fp32 [N]) the column sums of dx are accumulated into it in the same pass."""
    assert dy.is_contiguous() and pre.is_contiguous()
    dx = torch.empty_like(dy)
    if colsum_out is not None:
        N = dy.shape[-1]
        assert colsum_out.dtype == torch.float32 and colsum_out.numel() == N and colsum_out.is_contiguous()
        _call("dvla_act_bwd_colsum", dy.data_ptr(), pre.data_ptr(), dx.data_ptr(), dy.numel() // N, N, act,
              colsum_out.data_ptr(), _stream())
        return dx
    _call("dvla_act_bwd", dy.data_ptr(), pre.data_ptr(), dx.data_ptr(), dy.numel(), act, _stream())
    return dx


def mse_loss(pred2d, label2d, row_mask, weight, loss_out, dpred):
    rows, Cc = pred2d.shape
    assert pred2d.is_contiguous() and label2d.is_contiguous()
    _call("dvla_mse_loss", pred2d.data_ptr(), label2d.data_ptr(), _ptr(row_mask), rows, Cc, weight, loss_out.data_ptr(),
          _ptr(dpred), _stream())


def cosine_loss(pred2d, label2d, weight, loss_out, dpred):
    rows, Cc = pred2d.shape
    assert pred2d.is_contiguous() and label2d.is_contiguous()
    _call("dvla_cosine_loss", pred2d.data_ptr(), label2d.data_ptr(), rows, Cc, weight, loss_out.data_ptr(), _ptr(dpred),
          _stream())


def silog_loss(pred, label, lambd, weight, loss_out, dpred):
    assert pred.is_contiguous() and label.is_contiguous()
    n = pred.numel()
    stats = torch.zeros(load().dvla_silog_workspace_bytes() // 4, device=pred.device, dtype=torch.float32)
    _call("dvla_silog_stats", pred.data_ptr(), label.data_ptr(), n, stats.data_ptr(), _stream())
    _call("dvla_silog_finish", pred.data_ptr(), label.data_ptr(), n, stats.data_ptr(), lambd, weight, loss_out.data_ptr(),
          _ptr(dpred), _stream())


def sumsq(g_bf16, out_f32):
    _call("dvla_sumsq", g_bf16.data_ptr(), g_bf16.numel(), out_f32.data_ptr(), _stream())


def adamw(p, g, m, v, *, sumsq_t, lr_t, step_t, beta1, beta2, eps, weight_decay, max_norm, grad_scale=1.0,
          zero_grad=True):
    a = AdamWArgs(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), _ptr(sumsq_t), lr_t.data_ptr(),
                  step_t.data_ptr(), beta1, beta2, eps, weight_decay, max_norm, grad_scale, int(zero_grad))
    _call("dvla_adamw", C.byref(a), _stream())


def adamw_master(p32, p, g, m, v, *, sumsq_t, lr_t, step_t, beta1, beta2, eps, weight_decay, max_norm, grad_scale=1.0,
                 zero_grad=True):
    """`adamw` on fp32 master weights `p32`; the bf16 working copy `p` is overwritten with p32 rounded to bf16."""
    _need_cuda(p32, p, g, m, v)
    assert p32.dtype == torch.float32 and p.dtype == torch.bfloat16 and p32.numel() == p.numel() == g.numel() == m.numel()
    a = AdamWMasterArgs(p32.data_ptr(), p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p32.numel(), _ptr(sumsq_t),
                        lr_t.data_ptr(), step_t.data_ptr(), beta1, beta2, eps, weight_decay, max_norm, grad_scale,
                        int(zero_grad))
    _call("dvla_adamw_master", C.byref(a), _stream())


def grad_clip_scale(g, sumsq_t, max_norm, grad_scale=1.0):
    """g *= grad_scale * min(1, max_norm / (sqrt(sumsq) * grad_scale + 1e-6)) in place (clip_grad_norm_ on the flat buffer)."""
    _call("dvla_grad_clip_scale", g.data_ptr(), g.numel(), sumsq_t.data_ptr(), max_norm, grad_scale, _stream())


def set_sm_budget(n_sms: int) -> int:
    """SMs the persistent GEMM and attention-backward kernels size their grids for (0 = all); returns the previous value."""
    return load().dvla_set_sm_budget(int(n_sms))


def cat_broadcast(e, m):
    """e [n, a, C], m [b, C] (bf16, contiguous) -> [n, a + b, C] with m appended to every sequence."""
    _need_cuda(e, m)
    n, a, Cc = e.shape
    b = m.shape[0]
    assert e.is_contiguous() and m.is_contiguous() and m.shape[1] == Cc and e.dtype == m.dtype == torch.bfloat16
    out = torch.empty((n, a + b, Cc), device=e.device, dtype=torch.bfloat16)
    _call("dvla_cat_broadcast", e.data_ptr(), m.data_ptr(), out.data_ptr(), n, a, b, Cc, _stream())
    return out


def _dit_sampler_call(net, z, noise, n_steps, cfg_scale, fill):
    """Sets up dvla_dit_sampler_args for `net` (models.action_model.models.DiT) on condition rows z bf16 [bs, T, token] and the
    start state noise fp32 [bs, T, C], lets `fill(args)` set the integrator's fields, launches; -> fp32 [bs, T, C]."""
    _need_cuda(z, noise)
    bs, T, token = z.shape
    Cc = noise.shape[-1]
    H = net.x_embedder.linear.weight.shape[0]
    mlp = net.blocks[0].mlp.fc1.weight.shape[0]
    blocks = (DitBlockWeights * len(net.blocks))()
    for i, b in enumerate(net.blocks):
        blocks[i] = DitBlockWeights(b.attn.qkv.weight.data_ptr(), b.attn.qkv.bias.data_ptr(), b.attn.proj.weight.data_ptr(),
                                    b.attn.proj.bias.data_ptr(), b.mlp.fc1.weight.data_ptr(), b.mlp.fc1.bias.data_ptr(),
                                    b.mlp.fc2.weight.data_ptr(), b.mlp.fc2.bias.data_ptr())
    z = z.contiguous()
    noise = noise.contiguous().float()
    out = torch.empty((bs, T, Cc), device=z.device, dtype=torch.float32)
    ws_bytes = load().dvla_dit_sampler_workspace_bytes(bs, T, H, mlp, n_steps)
    ws = torch.empty(ws_bytes, device=z.device, dtype=torch.uint8)
    a = DitSamplerArgs()
    a.blocks = blocks
    a.depth, a.hidden, a.heads, a.mlp, a.token = len(net.blocks), H, net.num_heads, mlp, token
    a.freq, a.channels, a.T, a.batch = net.t_embedder.frequency_embedding_size, Cc, T, bs
    a.x_w, a.x_b = net.x_embedder.linear.weight.data_ptr(), net.x_embedder.linear.bias.data_ptr()
    a.t0_w, a.t0_b = net.t_embedder.mlp[0].weight.data_ptr(), net.t_embedder.mlp[0].bias.data_ptr()
    a.t2_w, a.t2_b = net.t_embedder.mlp[2].weight.data_ptr(), net.t_embedder.mlp[2].bias.data_ptr()
    a.z_w, a.z_b = net.z_embedder.linear.weight.data_ptr(), net.z_embedder.linear.bias.data_ptr()
    a.uncondition, a.pos = net.z_embedder.uncondition.data_ptr(), net.positional_embedding.data_ptr()
    a.final_w, a.final_b = net.final_layer.linear.weight.data_ptr(), net.final_layer.linear.bias.data_ptr()
    a.z, a.noise, a.out = z.data_ptr(), noise.data_ptr(), out.data_ptr()
    a.n_steps, a.cfg_scale = n_steps, float(cfg_scale)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
    fill(a)
    _call("dvla_dit_ddim_sample", C.byref(a), _stream())
    return out


def dit_ddim_sample(net, diffusion, z, noise, cfg_scale):
    """Fused DDIM sampler of the DiT action head (dit_sampler.cu): z bf16 [bs, T, token] condition rows, noise fp32 [bs, T, C]
    -> fp32 [bs, T, C].  `net` is models.action_model.models.DiT, `diffusion` the respaced SpacedDiffusion."""
    n_steps = diffusion.num_timesteps

    def fill(a):
        f32arr = lambda v: (_f32 * n_steps)(*[float(x) for x in v])     # noqa: E731
        a.timestep_map = (_i32 * n_steps)(*[int(t) for t in diffusion.timestep_map])
        a.sqrt_recip_alphas_cumprod = f32arr(diffusion.sqrt_recip_alphas_cumprod)
        a.sqrt_recipm1_alphas_cumprod = f32arr(diffusion.sqrt_recipm1_alphas_cumprod)
        a.alphas_cumprod_prev = f32arr(diffusion.alphas_cumprod_prev)
        a.integrator = DIT_DDIM
    return _dit_sampler_call(net, z, noise, n_steps, cfg_scale, fill)


def fm_t_values(n_steps):
    """The DiT timestep input of each flow-matching step, in execution order: fp32 i / n_steps, i = 0 .. n_steps-1, divided
    in fp32 as FMDiffusion.ddim_sample_loop's `torch.full((n,), float(i)) / T` (gaussian_diffusion.py:169) divides.  (On a
    CUDA tensor torch computes that division as a multiply by the fp32 reciprocal, one ulp off at i = 9 of 10: 0.90000004
    against 0.89999998 -- far below the bf16 rounding of the frequency features the value feeds.)"""
    return [float(v) for v in torch.arange(n_steps, dtype=torch.float32) / n_steps]


def dit_fm_sample(net, diffusion, z, start):
    """Fused flow-matching sampler of the DiT action head (`--use_fm`; dit_sampler.cu with the Euler integrator): z bf16
    [bs, T, token] condition rows, start fp32 [bs, T, C] start state -> fp32 [bs, T, C], as FMDiffusion.ddim_sample_loop
    (`diffusion`) computes the first half of its [2 bs, ...] state: guidance scale 1.0 over both branches, num_timesteps Euler
    steps of 1 / num_timesteps."""
    n_steps = diffusion.num_timesteps

    def fill(a):
        a.t_values = (_f32 * n_steps)(*fm_t_values(n_steps))
        a.integrator = DIT_FM_EULER
    return _dit_sampler_call(net, z, start, n_steps, 1.0, fill)
