"""ctypes binding of libaf3b200.so (C ABI declared in include/af3b200.h).

There is no CPU fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_PKG = Path(__file__).resolve().parent
_LIB_PATH = _PKG / "libaf3b200.so"

EPI_BIAS, EPI_GELU, EPI_RESID, EPI_SWIGLU, EPI_F32OUT, EPI_SWIGLU_CONCAT = 1, 2, 4, 8, 16, 64

_p, _i, _f, _i64, _sz = C.c_void_p, C.c_int, C.c_float, C.c_int64, C.c_size_t

# name -> (restype, argtypes); mirrors include/af3b200.h one to one (tests check every symbol resolves)
SIGNATURES = {
    "af3_last_error": (C.c_char_p, []),
    "af3_abi_version": (_i, []),
    "af3_set_pdl": (None, [_i]),
    "af3_trace_slot_bytes": (_sz, []),
    "af3_trace_begin": (_i, [_p, _sz]),
    "af3_trace_end": (_i, []),
    "af3_trace_seq": (_i, []),
    "af3_gemm_bf16": (_i, [_p, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p, _p, _i, _i]),
    "af3_gemm_workspace_bytes": (_sz, []),
    "af3_gemm_bf16_ws": (_i, [_p, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p, _p, _i, _i, _p, _sz]),
    "af3_pack_gate_up": (_i, [_p, _p, _p, _p, _i, _i]),
    "af3_logmel": (_i, [_p, _p, _i, _i, _p, _p, _p, _p, _p, _p, _p]),
    "af3_im2col_conv1": (_i, [_p, _p, _i, _p, _i, _i, _i]),
    "af3_im2col_conv2": (_i, [_p, _p, _p, _i, _i, _i]),
    "af3_layernorm": (_i, [_p, _p, _p, _p, _p, _i, _i, _f]),
    "af3_avgpool_layernorm": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _f]),
    "af3_rmsnorm": (_i, [_p, _p, _p, _p, _i, _i, _f, _p]),
    "af3_attention": (_i, [_p, _p, _i, _p, _p, _i, _i, _i, _p, _i, _i, _i, _i, _i, _i, _i, _f, _i, _p, _p]),
    "af3_rope_kv_append": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p]),
    "af3_rotary_time_emb": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _f, _f]),
    "af3_rope_table": (_i, [_p, _p, _i, _i, _p, _p, _p]),
    "af3_gated_residual": (_i, [_p, _p, _p, _p, _i, _p, _p, _i, _i]),
    "af3_gemm_qkv_rope": (_i, [_p, _p, _i, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _p, _p, _p, _i, _p, _p, _sz]),
    "af3_decode_attention": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _f]),
    "af3_decode_attention_scratch_bytes": (_sz, [_i, _i, _i, _i]),
    "af3_embed_scatter": (_i, [_p, _p, _i, _p, _i, _i64, _p, _i, _i, _p, _p, _p, _p]),
    "af3_argmax_scratch_bytes": (_sz, [_i]),
    "af3_argmax": (_i, [_p, _p, _i, _i, _p, _p]),
    "af3_logits_process_scratch_bytes": (_sz, [_i, _i]),
    "af3_logits_process_argmax": (_i, [_p, _p, _i, _i, _p, _p, _i, _p, _p, _p, _i, _p, _p, _p]),
    "af3_token_step": (_i, [_p, _p, _i, _p, _p, _p, _p, _i, _p, _p, _p]),
    "af3_quant_fp8": (_i, [_p, _p, _i, _p, _p, _i, _i]),
    "af3_gemm_fp8": (_i, [_p, _p, _i, _p, _p, _i, _p, _p, _i, _i, _i, _i, _i, _p, _p, _i, _p, _sz]),
    "af3_lm_head_xent_scratch_bytes": (_sz, [_i, _i]),
    "af3_lm_head_xent": (_i, [_p, _p, _i, _p, _i, _i, _i, _i, _p, _i64, _p, _i, _p, _p, _p]),
    "af3_gemm_qkv_rope_fp8": (_i, [_p, _p, _i, _p, _p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p, _p, _p, _i, _p, _p, _sz]),
}


_lib = None


class AF3Error(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load (once) and type the shared library.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise AF3Error(
            f"{_LIB_PATH} not found: build it with `python -m audio_flamingo_b200.build` "
            "(or __graft_entry__.build()); there is no CPU fallback for the AF3 hot path"
        )
    lib = C.CDLL(str(_LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = load().af3_last_error()
        raise AF3Error(f"{what}: {msg.decode() if msg else 'unknown error'} (status {status})")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
