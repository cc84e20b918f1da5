"""ctypes binding of libesvit_b200.so (the C ABI declared in include/esvit_b200.h).

There is no CPU / PyTorch fallback: if the library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_double, c_float, c_int, c_longlong, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libesvit_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(HERE), "include", "esvit_b200.h")

ERR_BAD_ARG = 1001

P, I, L, F, D = c_void_p, c_int, c_longlong, c_float, c_double

# name -> argtypes (restype is always int).  Keep in sync with include/esvit_b200.h
# (tests/test_abi.py parses the header and checks names + arity).
SIGNATURES = {
    "esvit_add_ln_fwd": [P, P, P, I, P, P, F, P, P, I, P, P, L, I, P],
    "esvit_add_ln_bwd": [P, I, P, P, P, P, P, P, I, P, P, P, P, P, L, I, P],
    "esvit_patch_merge_ln_fwd": [P, P, P, F, P, P, P, I, I, I, I, P],
    "esvit_patch_merge_ln_bwd": [P, P, P, P, P, P, P, P, I, I, I, I, P],
    "esvit_token_mean_fwd": [P, P, I, I, I, P],
    "esvit_token_mean_bwd": [P, P, P, I, I, I, P],
    "esvit_patch_embed_fwd": [P, P, P, P, P, F, P, P, P, I, I, I, I, P],
    "esvit_patch_embed_bwd": [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, P],
    "esvit_window_attn_expand_bias": [P, P, I, I, P],
    "esvit_window_attn_fwd": [P, P, P, P, I, P, P, I, I, I, I, I, I, I, F, P],
    "esvit_window_attn_bwd": [P, P, P, P, I, P, P, P, P, P, P, I, I, I, I, I, I, I, F, P],
    "esvit_window_attn_probs": [P, P, P, P, I, P, I, I, I, I, I, I, I, F, P],
    "esvit_gemm_bf16": [P, P, P, P, P, L, I, I, I, I, I, I, P],
    "esvit_gemm_mul_colsum2": [P, P, P, P, P, P, L, I, I, I, I, P],
    "esvit_gemm_f32": [P, P, P, P, L, I, I, I, P],
    "esvit_gemm_wgrad_ws_floats": [I, I],
    "esvit_gemm_wgrad": [P, P, P, P, L, I, I, I, I, P],
    "esvit_mlp_fwd": [P, P, P, P, P, P, P, P, L, I, P],
    "esvit_l2norm_fwd": [P, P, P, F, L, I, P],
    "esvit_l2norm_bwd": [P, P, P, P, L, I, P],
    "esvit_weight_norm_fwd": [P, P, P, P, L, I, P],
    "esvit_weight_norm_bwd": [P, P, P, P, P, P, L, I, P],
    "esvit_row_lse": [P, P, F, P, L, I, P],
    "esvit_dino_ce_fwd": [P, P, P, P, P, P, P, F, F, P, L, I, P],
    "esvit_dino_ce_bwd": [P, P, P, P, P, P, P, P, P, F, F, P, L, I, P],
    "esvit_weighted_sum": [P, P, I, P, P],
    "esvit_row_softmax_q_max_k": [],
    "esvit_row_softmax_q": [P, P, F, P, P, L, I, P],
    "esvit_dino_ce_q_fwd": [P, P, P, P, P, F, P, L, I, P],
    "esvit_dino_ce_q_bwd": [P, P, P, P, P, P, P, F, P, L, I, P],
    "esvit_mixup_q_kpad": [I],
    "esvit_mixup_q": [P, P, I, I, I, F, P, P, P, P],
    "esvit_colsum_workspace_rows": [],
    "esvit_colsum": [P, L, I, P, P, P],
    "esvit_center_ema": [P, P, F, D, P, I, P],
    "esvit_normalize_rows": [P, P, L, I, F, P],
    "esvit_region_match": [P, P, I, I, I, I, I, P, P, P],
    "esvit_mhsa_fwd": [P, P, P, I, I, I, I, F, P],
    "esvit_mhsa_bwd": [P, P, P, P, P, P, I, I, I, I, F, P],
    "esvit_conv_im2col": [P, P, I, I, I, I, I, I, I, I, I, P],
    "esvit_conv_col2im": [P, P, I, I, I, I, I, I, I, I, P],
    "esvit_mhsa_win_fwd": [P, P, P, I, I, I, I, I, I, F, P],
    "esvit_mhsa_win_bwd": [P, P, P, P, P, P, I, I, I, I, I, I, F, P],
    "esvit_dwbn_fwd_stats": [P, P, P, P, P, I, I, I, I, I, I, P],
    "esvit_dwbn_fwd_apply": [P, P, P, P, P, P, P, P, P, L, I, I, F, F, P],
    "esvit_dwbn_bwd_stats": [P, P, P, P, P, P, P, L, I, P],
    "esvit_dwbn_bwd_apply": [P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, I, P],
    "esvit_headbn_fwd_stats": [P, P, P, L, I, P],
    "esvit_headbn_fwd_apply": [P, P, P, P, P, P, P, P, P, L, I, I, F, F, P],
    "esvit_headbn_bwd_stats": [P, P, P, P, P, P, P, L, I, P],
    "esvit_headbn_bwd_apply": [P, P, P, P, P, P, P, P, L, I, I, P],
    "esvit_vil_sc_ws_floats": [I, I, I, I],
    "esvit_vil_sc_fwd": [P, P, P, P, P, P, P, P, I, I, I, I, F, P],
    "esvit_vil_sc_bwd": [P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, F, P],
    "esvit_vil_dense_parts": [I],
    "esvit_vil_dense_fwd": [P, P, P, P, I, I, I, I, F, P],
    "esvit_vil_dense_bwd": [P, P, P, P, P, P, P, P, P, I, I, I, I, F, P],
    "esvit_vil_im2col": [P, P, I, I, I, I, I, I, I, I, P],
    "esvit_vil_col2im": [P, P, I, I, I, I, I, I, I, I, P],
    "esvit_vil_cls_cat_fwd": [P, P, P, I, I, I, P],
    "esvit_vil_cls_cat_bwd": [P, P, P, I, I, I, I, P],
    "esvit_vil_bias_spmv": [P, P, P, P, P, P, I, I, P, I, P],
    "esvit_vit_patches": [P, P, I, I, I, P],
    "esvit_vit_tokens_fwd": [P, P, P, P, I, I, I, P],
    "esvit_vit_tokens_bwd": [P, P, P, P, P, I, I, I, I, P],
    "esvit_vit_split": [P, P, P, I, I, I, I, P],
    "esvit_ema_multi": [P, P, P, I, D, P],
    "esvit_clip_multi": [P, P, I, F, P, P, P],
    "esvit_grad_sumsq_multi": [P, P, I, P, P],
    "esvit_adamw_ema_multi": [P, P, P, P, P, P, P, P, I, P, P, P, P],
    "esvit_lars_sums_multi": [P, P, P, I, P, P],
    "esvit_sgd_ema_multi": [P, P, P, P, P, P, P, I, P, P, P, P],
    "esvit_knn_prep": [P, P, P, P, L, L, I, P],
    "esvit_knn_select": [P, L, P, P, P, P, P, I, I, I, I, I, P, P, P, P, P, P],
    "esvit_knn_vote": [P, P, P, P, L, I, F, I, P, P],
    "esvit_probe_ce": [P, I, P, I, I, P, P, P, P, P, P, P],
    "esvit_augment_coeffs": [P, P, P, I, I, P],
    "esvit_augment_resize_h": [P, P, P, P, P, I, L, P],
    "esvit_augment_color": [P, P, P, P, P, I, I, I, P],
    "esvit_augment_eval_coeffs": [P, P, P, I, I, P],
    "esvit_augment_eval_resize_h": [P, P, P, P, P, I, I, L, P],
    "esvit_augment_eval_resize_v": [P, P, P, P, P, I, I, P],
}

_lib = None


class EsvitKernelError(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """Load the shared library, failing loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise EsvitKernelError(
            f"{LIB_PATH} not found: the esvit_b200 CUDA library has not been built "
            "(run `python -m esvit_b200.build` or `__graft_entry__.build()`); there is no CPU fallback")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = c_int
    _lib = lib
    return lib


def _cuda_error_string(code: int) -> str:
    try:
        import torch
        return torch.cuda.cudart().cudaGetErrorString(code) if hasattr(torch.cuda.cudart(), "cudaGetErrorString") \
            else f"cudaError {code}"
    except Exception:
        return f"cudaError {code}"


def call(name: str, *args) -> None:
    """Invoke an entry point; non-zero status -> Python exception (the reference's error convention
    at this boundary is Python exceptions, SURVEY.md §8b)."""
    rc = getattr(load(), name)(*args)
    if rc != 0:
        if rc == ERR_BAD_ARG:
            raise ValueError(f"{name}: unsupported shape / argument (ESVIT_ERR_BAD_ARG)")
        raise EsvitKernelError(f"{name} failed: {_cuda_error_string(rc)} (status {rc})")


# ---- instrumentation used by bench.py (launch counting; live CUDA-event timing of one entry point) --------------
# kernels launched per call of each entry point (entries that launch more than one kernel are computed per call)
_LAUNCHES = {"esvit_colsum": 2, "esvit_gemm_mul_colsum2": 2, "esvit_gemm_wgrad": 2,
             "esvit_mixup_q": 2,  # GEMM + fold; mixup weights + product
             "esvit_probe_ce": 2,
             "esvit_headbn_fwd_stats": 2, "esvit_headbn_fwd_apply": 2, "esvit_headbn_bwd_stats": 2,
             "esvit_headbn_bwd_apply": 3}
_launch_count = 0
_timed_names = set()
_timed_events = []
# algorithmic-bytes meta per timed entry point (bench.py roofline): extracted from the call's own arguments
_META = {
    "esvit_dino_ce_bwd": lambda a: {"rows": int(a[-3]), "K": int(a[-2])},
    "esvit_window_attn_bwd": lambda a: _attn_meta(a),
    "esvit_window_attn_fwd": lambda a: _attn_meta(a),
    "esvit_window_attn_probs": lambda a: _attn_meta(a),
    "esvit_gemm_bf16": lambda a: {"M": int(a[5]), "N": int(a[6]), "K": int(a[7]), "b_mn": int(a[9]), "act": int(a[10]),
                                  "pre": a[4] is not None and a[4].value is not None},
    "esvit_gemm_mul_colsum2": lambda a: {"M": int(a[6]), "N": int(a[7]), "K": int(a[8])},
    "esvit_gemm_wgrad": lambda a: {"T": int(a[4]), "N": int(a[5]), "K": int(a[6])},
    "esvit_mlp_fwd": lambda a: {"M": int(a[8]), "C": int(a[9]), "student": a[6] is not None and a[6].value is not None},
    "esvit_add_ln_fwd": lambda a: {"T": int(a[-3]), "C": int(a[-2]), "has_x": a[0] is not None and a[0].value is not None,
                                   "has_delta": a[1] is not None and a[1].value is not None},
    "esvit_add_ln_bwd": lambda a: {"T": int(a[-3]), "C": int(a[-2])},
    "esvit_dino_ce_fwd": lambda a: {"rows": int(a[-3]), "K": int(a[-2])},
    "esvit_dino_ce_q_fwd": lambda a: {"rows": int(a[-3]), "K": int(a[-2])},
    "esvit_dino_ce_q_bwd": lambda a: {"rows": int(a[-3]), "K": int(a[-2])},
    "esvit_row_softmax_q": lambda a: {"rows": int(a[-3]), "K": int(a[-2])},
    "esvit_mixup_q": lambda a: {"ncrops": int(a[2]), "B": int(a[3]), "K": int(a[4])},
    "esvit_conv_im2col": lambda a: {"B": int(a[3]), "C": int(a[4]), "H": int(a[5]), "W": int(a[6]), "k": int(a[7]),
                                    "s": int(a[8]), "p": int(a[9]), "Kp": int(a[10])},
    "esvit_conv_col2im": lambda a: {"B": int(a[2]), "C": int(a[3]), "H": int(a[4]), "W": int(a[5]), "k": int(a[6]),
                                    "s": int(a[7]), "p": int(a[8]), "Kp": int(a[9])},
    "esvit_dwbn_fwd_stats": lambda a: {"B": int(a[5]), "H": int(a[6]), "W": int(a[7]), "Hp": int(a[8]), "Wp": int(a[9]),
                                       "C": int(a[10])},
    "esvit_dwbn_fwd_apply": lambda a: {"N": int(a[9]), "C": int(a[10])},
    "esvit_dwbn_bwd_stats": lambda a: {"N": int(a[7]), "C": int(a[8])},
    "esvit_headbn_fwd_stats": lambda a: {"N": int(a[3]), "C": int(a[4])},
    "esvit_headbn_fwd_apply": lambda a: {"N": int(a[9]), "C": int(a[10])},
    "esvit_headbn_bwd_stats": lambda a: {"N": int(a[7]), "C": int(a[8])},
    "esvit_headbn_bwd_apply": lambda a: {"N": int(a[8]), "C": int(a[9])},
    "esvit_dwbn_bwd_apply": lambda a: {"B": int(a[10]), "H": int(a[11]), "W": int(a[12]), "Hp": int(a[13]),
                                       "Wp": int(a[14]), "C": int(a[15])},
    "esvit_mhsa_win_fwd": lambda a: {"B": int(a[3]), "H": int(a[4]), "W": int(a[5]), "w": int(a[6]), "C": int(a[7]),
                                     "nH": int(a[8])},
    "esvit_mhsa_win_bwd": lambda a: {"B": int(a[6]), "H": int(a[7]), "W": int(a[8]), "w": int(a[9]), "C": int(a[10]),
                                     "nH": int(a[11])},
    "esvit_vil_sc_fwd": lambda a: {"B": int(a[8]), "nx": int(a[9]), "ny": int(a[10]), "nH": int(a[11])},
    "esvit_vil_sc_bwd": lambda a: {"B": int(a[15]), "nx": int(a[16]), "ny": int(a[17]), "nH": int(a[18])},
    "esvit_vil_dense_fwd": lambda a: {"B": int(a[4]), "L": int(a[5]), "C": int(a[6]), "nH": int(a[7])},
    "esvit_vil_dense_bwd": lambda a: {"B": int(a[9]), "L": int(a[10]), "C": int(a[11]), "nH": int(a[12])},
    "esvit_mhsa_fwd": lambda a: {"B": int(a[3]), "L": int(a[4]), "C": int(a[5]), "nH": int(a[6])},
    "esvit_mhsa_bwd": lambda a: {"B": int(a[6]), "L": int(a[7]), "C": int(a[8]), "nH": int(a[9])},
    "esvit_vit_tokens_bwd": lambda a: {"B": int(a[-5]), "N": int(a[-4]), "D": int(a[-3])},
    "esvit_patch_embed_fwd": lambda a: {"B": int(a[-5]), "H": int(a[-4]), "W": int(a[-3]), "E": int(a[-2])},
    "esvit_patch_embed_bwd": lambda a: {"B": int(a[-5]), "H": int(a[-4]), "W": int(a[-3]), "E": int(a[-2])},
}


def _attn_meta(a):
    """(..., B, H, W, C, nH, ws, shift, scale, stream) of the window-attention entry points"""
    B, H, W, C, nH, ws = (int(a[i]) for i in (-9, -8, -7, -6, -5, -4))
    return {"tokens": B * H * W, "C": C, "nH": nH, "ws": ws, "windows": B * (-(-H // ws)) * (-(-W // ws))}


def reset_counters() -> None:
    global _launch_count
    _launch_count = 0
    _timed_events.clear()


def launch_count() -> int:
    return _launch_count


def time_entry_point(names) -> None:
    """Bracket every call of the named entry point(s) with CUDA events on the launching (current) stream."""
    global _timed_names
    if names is None:
        _timed_names = set()
    elif isinstance(names, str):
        _timed_names = {names}
    else:
        _timed_names = set(names)


def timed_results():
    """[{name, ms, ...meta}] of the timed entry points (call after a device synchronize)."""
    out = []
    for name, e0, e1, meta in _timed_events:
        d = {"name": name, "ms": e0.elapsed_time(e1)}
        d.update(meta)
        out.append(d)
    return out


_plain_call = call


def call(name: str, *args) -> None:  # noqa: F811  (instrumented wrapper)
    global _launch_count
    if name == "esvit_ema_multi":
        _launch_count += (args[3] + 63) // 64
    elif name == "esvit_clip_multi":
        _launch_count += 2 * ((args[2] + 63) // 64)
    elif name == "esvit_grad_sumsq_multi":
        _launch_count += (args[2] + 63) // 64
    elif name == "esvit_lars_sums_multi":
        _launch_count += (args[3] + 63) // 64
    elif name == "esvit_adamw_ema_multi":
        _launch_count += (args[8] + 31) // 32 + 1
    elif name == "esvit_sgd_ema_multi":
        _launch_count += (args[7] + 31) // 32 + 1
    else:
        _launch_count += _LAUNCHES.get(name, 1)
    if name in _timed_names:
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _plain_call(name, *args)
        e1.record()
        _timed_events.append((name, e0, e1, _META[name](args) if name in _META else {}))
    else:
        _plain_call(name, *args)
