"""ctypes binding of libslamkit_b200.so (the C ABI declared in include/slamkit_b200.h).

There is no fallback: if the shared library is missing, or a compute entry point is called without a CUDA device,
the call raises.  PyTorch is used only to own device memory and streams; every pointer crossing this boundary is a
raw device address.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Dict, List, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libslamkit_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "slamkit_b200.h")

_lib: Optional[C.CDLL] = None


class SkError(RuntimeError):
    pass


class SkLmConfig(C.Structure):
    _fields_ = [
        ("vocab_size", C.c_int32),
        ("hidden", C.c_int32),
        ("n_layers", C.c_int32),
        ("n_heads", C.c_int32),
        ("n_kv_heads", C.c_int32),
        ("head_dim", C.c_int32),
        ("ffn", C.c_int32),
        ("max_positions", C.c_int32),
        ("rms_eps", C.c_float),
        ("tie_embeddings", C.c_int32),
        ("qkv_bias", C.c_int32),
    ]


class SkOptConfig(C.Structure):
    _fields_ = [
        ("vocab_size", C.c_int32),
        ("hidden", C.c_int32),
        ("n_layers", C.c_int32),
        ("n_heads", C.c_int32),
        ("ffn", C.c_int32),
        ("max_positions", C.c_int32),
        ("ln_eps", C.c_float),
        ("tie_embeddings", C.c_int32),
        ("post_ln", C.c_int32),
        ("proj_dim", C.c_int32),
    ]


class SkNeoxConfig(C.Structure):
    _fields_ = [
        ("vocab_size", C.c_int32),
        ("hidden", C.c_int32),
        ("n_layers", C.c_int32),
        ("n_heads", C.c_int32),
        ("ffn", C.c_int32),
        ("max_positions", C.c_int32),
        ("rot_dims", C.c_int32),
        ("ln_eps", C.c_float),
    ]


class SkHubertConfig(C.Structure):
    _fields_ = [
        ("n_conv", C.c_int32),
        ("conv_dim", C.c_int32),
        ("conv_kernel", C.c_int32 * 8),
        ("conv_stride", C.c_int32 * 8),
        ("hidden", C.c_int32),
        ("n_heads", C.c_int32),
        ("ffn", C.c_int32),
        ("n_layers", C.c_int32),
        ("pos_conv_kernel", C.c_int32),
        ("pos_conv_groups", C.c_int32),
        ("n_units", C.c_int32),
        ("ln_eps", C.c_float),
        ("pad", C.c_int32),
    ]


class SkSampling(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64),
        ("top_p", C.c_double),
        ("temperature", C.c_float),
        ("do_sample", C.c_int32),
        ("top_k", C.c_int32),
        ("n_eos", C.c_int32),
        ("eos", C.c_int32 * 8),
        ("pad_token_id", C.c_int32),
        ("max_length", C.c_int32),
    ]


class SkDecodeState(C.Structure):
    _fields_ = [
        ("tokens", C.c_void_p),
        ("pos", C.c_void_p),
        ("finished", C.c_void_p),
        ("n_gen", C.c_void_p),
        ("out", C.c_void_p),
        ("step", C.c_void_p),
        ("max_new", C.c_int32),
        ("reserved", C.c_int32),
    ]


class SkLogitRules(C.Structure):
    _fields_ = [
        ("history", C.c_void_p),
        ("presence", C.c_void_p),
        ("scratch", C.c_void_p),
        ("penalty", C.c_float),
        ("ngram", C.c_int32),
        ("min_step", C.c_int32),
        ("prompt_len", C.c_int32),
        ("hist_ld", C.c_int32),
        ("reserved", C.c_int32),
    ]


class SkGemmPlan(C.Structure):
    _fields_ = [
        ("bn", C.c_int32),
        ("epi_warps", C.c_int32),
        ("splits", C.c_int32),
        ("sk_units", C.c_int32),
        ("sk_groups", C.c_int32),
        ("sk_G", C.c_int32),
        ("sk_colunits", C.c_int32),
        ("tma_store", C.c_int32),
        ("grid", C.c_int32),
    ]


class SkGemmSplitDesc(C.Structure):
    """sk_gemm_split / sk_gemm_split_plan: the batched, split-bf16 GEMM of the HuBERT path (see the header)."""
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("batch", C.c_int32), ("a_mode", C.c_int32),
        ("passes", C.c_int32),
        ("A", C.c_void_p), ("A_lo", C.c_void_p), ("lda", C.c_int32), ("a_mn", C.c_int32),
        ("a_inner", C.c_int64), ("a_rows", C.c_int64), ("a_row_stride", C.c_int64), ("a_batch_stride", C.c_int64),
        ("B", C.c_void_p), ("B_lo", C.c_void_p), ("ldb", C.c_int32),
        ("C", C.c_void_p), ("C_lo", C.c_void_p), ("ldc", C.c_int32), ("out_f32", C.c_int32),
        ("bias", C.c_void_p), ("bias_f32", C.c_int32),
        ("residual", C.c_void_p), ("residual_lo", C.c_void_p), ("ldr", C.c_int32), ("act", C.c_int32),
        ("col_gin", C.c_int32), ("col_gout", C.c_int32), ("force_bn", C.c_int32),
    ]


def declared_symbols() -> List[str]:
    """Names of all functions declared in include/slamkit_b200.h (used by the CPU symbol-export test)."""
    text = open(HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sk_[a-z0-9_]+)\s*\(", text)))


def load() -> C.CDLL:
    """Load the shared library (no CUDA call is made here, so this works on a CPU-only box)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SkError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C slamkit_b200/csrc`). slamkit_b200 has no CPU or PyTorch fallback."
        )
    lib = C.CDLL(LIB_PATH)
    lib.sk_last_error.restype = C.c_char_p
    for name in ("sk_lm_param_count", "sk_lm_workspace_bytes", "sk_launch_count", "sk_hubert_param_count", "sk_hubert_prepared_bytes",
                 "sk_hubert_workspace_bytes", "sk_gemm_ws_bytes", "sk_lm_kv_cache_bytes", "sk_lm_decode_workspace_bytes",
                 "sk_attn_decode_partial_bytes", "sk_vocoder_param_count", "sk_vocoder_prepared_bytes",
                 "sk_vocoder_workspace_bytes", "sk_lm_fp32_prepared_bytes"):
        if hasattr(lib, name):
            getattr(lib, name).restype = C.c_int64
    for name in ("sk_lm_logits", "sk_lm_logits_f32"):
        getattr(lib, name).restype = C.c_void_p
    lib.sk_lm_destroy.restype = None
    _p, _i = C.c_void_p, C.c_int
    for name in ("sk_select_next_ex", "sk_select_next_ex_f32"):
        getattr(lib, name).argtypes = [_p, _i, _i, _i, _p, C.POINTER(SkSampling), _p, C.POINTER(SkDecodeState),
                                       C.POINTER(SkLogitRules), _p]
    lib.sk_presence_init.argtypes = [_p, _i, _i, _i, _i, _p, _p]
    lib.sk_lm_kv_fanout.argtypes = [_p, _p, _i, _i, _p, _i, _p, _p]
    if hasattr(lib, "sk_hubert_destroy"):
        lib.sk_hubert_destroy.restype = None
    if hasattr(lib, "sk_vocoder_destroy"):
        lib.sk_vocoder_destroy.restype = None
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise SkError(f"slamkit_b200 error {rc}: {load().sk_last_error().decode()}")


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise SkError("slamkit_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    lib = load()
    cc = lib.sk_device_cc()
    if cc != 90:
        raise SkError(f"slamkit_b200 kernels are built for sm_90a only; current device reports compute capability {cc}")
    return lib


def ptr(t) -> C.c_void_p:
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return C.c_void_p(0)
    return C.c_void_p(t.data_ptr())


def stream_ptr() -> C.c_void_p:
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def f32(x: float) -> C.c_float:
    return C.c_float(float(x))
