"""ctypes binding of libb200attn.so (include/b200_paged_attn.h).

This is the only door to the GPU kernels.  There is no CPU fallback: if the
shared library is missing or a call fails, the product raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent.parent / "lib" / "libb200attn.so"

# name -> (restype, argtypes); mirrors include/b200_paged_attn.h one to one
_vp, _i, _i64, _f, _sz, _u64 = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t, C.c_uint64
SIGNATURES = {
    "b200_init": (_i, [_i, C.POINTER(_vp)]),
    "b200_destroy": (None, [_vp]),
    "b200_strerror": (C.c_char_p, [_i]),
    "b200_last_cuda_error": (C.c_char_p, [_vp]),
    "b200_sm_count": (_i, [_vp]),
    "b200_abi_version": (_i, []),
    "b200_set_pdl": (_i, [_i]),
    "b200_kv_bind": (_i, [_vp, _vp, _vp, _i, _i64, _i, _i, _i]),
    "b200_kv_bind_fp8": (_i, [_vp, _vp, _vp, _i, _i64, _i, _i, _i, _f, _f]),
    "b200_kv_gather": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i64, _vp, _i64, _i, _vp]),
    "b200_decode_workspace_bytes": (_sz, [_vp, _i, _i]),
    "b200_store_kv": (_i, [_vp, _i, _vp, _i64, _vp, _i64, _vp, _i, _vp]),
    "b200_paged_decode": (_i, [_vp, _i, _vp, _i64, _vp, _i, _vp, _vp, _i64, _i, _i, _f, _vp, _sz, _vp]),
    "b200_paged_decode_fused": (_i, [_vp, _i, _vp, _i64, _vp, _vp, _vp, _f, _vp, _i, _vp, _vp, _i64, _i, _i, _f, _vp, _sz, _vp]),
    "b200_paged_prefill": (_i, [_vp, _i, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i, _vp, _i64,
                                 _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_prefill_packed_kv": (_i, [_vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_rmsnorm": (_i, [_vp, _i64, _vp, _vp, _i64, _i, _i, _f, _vp]),
    "b200_add_rmsnorm": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "b200_qknorm_rope_store": (_i, [_vp, _i, _vp, _i64, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _i, _vp]),
    "b200_allreduce_add_rmsnorm": (_i, [_vp, _u64, _u64, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "b200_allreduce_add_rmsnorm_nvls": (_i, [_vp, _vp, _u64, _u64, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "b200_silu_mul": (_i, [_vp, _vp, _i, _i, _vp]),
    "b200_embedding": (_i, [_vp, _vp, _vp, _i, _i, _i64, _vp]),
    "b200_gather_tokens": (_i, [_vp, _vp, _vp, _i, _vp]),
    "b200_sample": (_i, [_vp, _i, _i64, _vp, _i, _i, _i64, _u64, _u64, _vp, _vp, _vp, _vp]),
    "b200_sample_filter_workspace_words": (_i64, [_i]),
    "b200_sample_filter_stage": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "b200_sample_filtered": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _i, _i, _i64, _u64, _u64, _vp, _vp, _vp, _vp, _vp]),
    # decode-size projections on wgmma (csrc/linear_tc.cu) and the fused LM head / layer tail experiments
    "b200_linear": (_i, [_vp, _i64, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_add_rmsnorm_partials": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _f, _i, _vp]),
    "b200_lm_head_sample": (_i, [_vp, _i64, _vp, _i, _i, _i, _vp, _i64, _u64, _u64, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b200_layer_tail_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "b200_layer_tail": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _sz, _i, _i, _i, _i, _f, _i, _i, _vp]),
}

_lib = None


class B200Error(RuntimeError):
    pass


def lib_path() -> Path:
    return Path(os.environ.get("B200ATTN_LIB", _LIB_PATH))


def load():
    """dlopen the library and type every exported symbol.  Raises if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not path.exists():
        raise B200Error(
            f"{path} not found: build it with `make -C nano-vllm_b200/csrc` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback.")
    lib = C.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the header and the library diverge
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int, ctx=None):
    if code == 0:
        return
    lib = load()
    msg = lib.b200_strerror(code).decode()
    if code == -3:                        # ctx None: the text of this thread's last context-less call
        msg += ": " + lib.b200_last_cuda_error(ctx).decode()
    raise B200Error(f"libb200attn: {msg} (code {code})")


class Handle:
    """One b200_ctx per process (one process per GPU)."""

    def __init__(self, device: int):
        self.lib = load()
        h = _vp()
        check(self.lib.b200_init(device, C.byref(h)))
        self.ptr = h
        self.sm_count = self.lib.b200_sm_count(h)
        self.kv = None            # keeps the bound cache tensors alive
        self.workspace = None

    def close(self):
        if self.ptr:
            self.lib.b200_destroy(self.ptr)
            self.ptr = None


_handle: Handle | None = None


def handle(device: int | None = None) -> Handle:
    """Process-wide handle; created on first use for the current CUDA device."""
    global _handle
    if _handle is None:
        import torch
        if not torch.cuda.is_available():
            raise B200Error("no CUDA device: the GPU path has no CPU fallback")
        _handle = Handle(torch.cuda.current_device() if device is None else device)
    return _handle


def reset_handle():
    global _handle
    if _handle is not None:
        _handle.close()
    _handle = None
