"""ctypes binding of libmidi_b200.so (C ABI in include/midi_b200.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.
Tensors cross the boundary as raw device pointers (`tensor.data_ptr()`) plus sizes and the
current CUDA stream handle; PyTorch is only the allocator / stream provider.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmidi_b200.so")

vp, i32, i64, f32, sz, u64 = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_size_t, C.c_ulonglong

# name -> (restype, argtypes).  Mirrors include/midi_b200.h one to one.
SIGNATURES = {
    "b200_last_error": (C.c_char_p, []),
    "b200_abi_version": (i32, []),
    "b200_launch_count": (i64, []),
    "b200_device_info": (i32, [vp, vp, vp]),
    "b200_embed_sum_fwd": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "b200_inner_input_fwd": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "b200_inner_input_bwd_hidden": (i32, [vp, vp, i32, i32, i32, vp]),
    "b200_inner_input_rows_fwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "b200_inner_input_rows_bwd_hidden": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "b200_batch_to_xy_i16": (i32, [vp, i32, i32, i32, vp, vp, vp]),
    "b200_batch_to_xy_packed_i16": (i32, [vp, i32, vp, i32, i32, vp, vp, vp]),
    "b200_augment_i16": (i32, [vp, i32, i32, i32, vp, vp, vp]),
    "b200_embed_bwd_workspace_bytes": (sz, [i32, i32, i32]),
    "b200_embed_bwd": (i32, [vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp, sz, vp]),
    "b200_rmsnorm_fwd": (i32, [vp, vp, vp, vp, i32, i32, f32, vp]),
    "b200_add_rmsnorm_fwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, f32, vp]),
    "b200_rmsnorm_bwd_parts": (i32, []),
    "b200_rmsnorm_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, sz, vp]),
    "b200_rope_table": (i32, [vp, i32, i32, i32, vp, vp, vp, vp]),
    "b200_rope_qk": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp]),
    "b200_rope_qk_seg": (i32, [vp, vp, vp, i32, vp, i32, i32, i32, i32, vp]),
    "b200_rope_qk_ragged": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
    "b200_swiglu_fwd": (i32, [vp, vp, i64, i32, vp]),
    "b200_swiglu_bwd": (i32, [vp, vp, vp, i64, i32, vp]),
    "b200_scale_bf16": (i32, [vp, vp, i64, f32, vp]),
    "b200_gemm_workspace_bytes": (sz, [i32, i32, i32]),
    "b200_gemm_tail_workspace_bytes": (sz, [i32, i32, i32, i32]),
    "b200_gemm_suggest_splits": (i32, [i32, i32, i32, i32]),
    "b200_gemm_plan": (i32, [i32, i32, i32, i32, vp, vp]),
    "b200_gemm_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, sz, vp]),
    "b200_gemm_bf16_rope": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, vp]),
    "b200_gemm_bf16_rope_seg": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp]),
    "b200_gemm_bf16_swiglu": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b200_attn_causal_fwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp]),
    "b200_attn_causal_fwd_wgmma": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp]),
    "b200_attn_causal_bwd_wgmma": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp, vp, vp]),
    "b200_attn_causal_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp, vp, vp]),
    "b200_attn_causal_fwd_seg_wgmma": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, vp, vp, vp]),
    "b200_attn_causal_bwd_seg_wgmma": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, vp, vp, vp, vp, vp]),
    "b200_attn_tiny_fwd": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, f32, vp, vp, vp]),
    "b200_attn_tiny_bwd": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp, vp, vp]),
    "b200_ce_fwd": (i32, [vp, vp, vp, vp, vp, i64, i32, i32, i64, vp]),
    "b200_ce_bwd": (i32, [vp, vp, vp, vp, i64, i32, i32, i64, f32, vp, i32, vp]),
    "b200_argmax_hits_parts": (i32, []),
    "b200_argmax_hits": (i32, [vp, vp, i64, i32, i32, i64, vp, vp, sz, vp]),
    "b200_gradnorm_parts": (i32, []),
    "b200_grad_clip_coef": (i32, [vp, i64, f32, vp, vp, sz, vp]),
    "b200_adamw_step": (i32, [vp, vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, i32, vp, vp]),
    "b200_gemv_bf16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b200_gemv_fused": (i32, [vp, vp, i32, vp, i32, vp, f32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b200_attn_decode_fused": (i32, [vp, vp, vp, vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp, i32, i32, i32, f32, i32, vp, sz, vp]),
    "b200_kv_append": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]),
    "b200_attn_decode_workspace_bytes": (sz, [i32, i32, i32, i32]),
    "b200_attn_decode": (i32, [vp, vp, vp, vp, i32, i32, vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, f32, i32, vp, sz, vp]),
    "b200_sample_topp_topk": (i32, [vp, i32, i32, i32, i32, f32, i32, vp, vp, vp]),
    "b200_sample_from_logits": (i32, [vp, i32, i32, i32, f32, f32, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, i32, vp]),
    "b200_uniform_fill": (i32, [vp, i32, u64, vp, vp]),
    "b200_event_commit": (i32, [vp, vp, vp, vp, i32, i32, i32, vp]),
    "b200_kv_append_ragged": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp, vp]),
    "b200_attn_decode_ragged": (i32, [vp, vp, vp, vp, i32, i32, vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, f32, i32, vp, sz,
                                      vp, vp]),
    "b200_attn_decode_fused_ragged": (i32, [vp, vp, vp, vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp, i32, i32, i32, f32, i32,
                                            vp, sz, vp, vp]),
    "b200_event_commit_ragged": (i32, [vp, vp, vp, vp, i32, i32, i32, vp, vp]),
    "b200_event_commit_queue": (i32, [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, i32, vp]),
    "b200_sample_from_logits_rows": (i32, [vp, i32, i32, i32, vp, vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, vp, i32, vp]),
    "b200_uniform_fill_rows": (i32, [vp, i32, vp, vp, vp, vp, i32, vp]),
    "b200_decode_desc_bytes": (sz, []),
    "b200_decode_events_workspace_bytes": (sz, [vp]),
    "b200_decode_events": (i32, [vp, i32, vp, sz, vp]),
    "b200_decode_events_ragged": (i32, [vp, vp, i32, vp, sz, vp]),
    "b200_decode_events_queue": (i32, [vp, vp, vp, vp, i32, i32, vp, sz, vp]),
    "b200_decode_events_queue_rows": (i32, [vp, vp, vp, vp, i32, i32, vp, sz, vp, vp, vp, vp, vp, vp]),
    "b200_decode_events_queue_stream": (i32, [vp, vp, vp, vp, i32, i32, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
}


class DecodeDesc(C.Structure):
    """b200_decode_desc of include/midi_b200.h (field for field)."""
    _fields_ = [("outer_w", vp), ("inner_w", vp), ("n_outer", i32), ("n_inner", i32),
                ("outer_norm", vp), ("inner_norm", vp), ("lm_head", vp), ("emb_outer", vp), ("emb_inner", vp),
                ("H", i32), ("I_outer", i32), ("I_inner", i32), ("nh_outer", i32), ("nh_inner", i32), ("V", i32), ("pitch", i32),
                ("eps", f32),
                ("kv_outer", vp), ("block_table", vp), ("max_pages", i32), ("page", i32),
                ("cos_outer", vp), ("sin_outer", vp), ("cos_inner", vp), ("sin_inner", vp),
                ("pos", vp), ("ev_in", vp), ("seq", vp), ("max_len", i32),
                ("rng_state", vp), ("dense_mask", vp), ("lut", vp),
                ("n_event_types", i32), ("eos_id", i32), ("pad_id", i32),
                ("temp", f32), ("top_p", f32), ("top_k", i32), ("batch", i32), ("prof", vp)]


AUG_SKIP, AUG_PITCH, AUG_VELOCITY, AUG_CC_VALUE, AUG_BPM, AUG_CHANNEL, AUG_DRUM, AUG_COLS = 0, 1, 2, 3, 4, 5, 6, 10


class AugmentIds(C.Structure):
    """b200_augment_ids of include/midi_b200.h (field for field): event ids and the first id of each parameter."""
    _fields_ = [(n, i32) for n in ("note", "patch_change", "control_change", "set_tempo", "key_signature", "track",
                                   "channel", "pitch", "velocity", "controller", "value", "bpm", "sf", "mi")]


class B200Error(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()
launch_count = 0   # number of C-ABI compute calls issued (bench.py reports kernel launches from this)


def load() -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built -- there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise B200Error(f"{LIB_PATH} not found: build it with `python midi-model_b200/build_ext.py` "
                            "(or __graft_entry__.build()).  There is no CPU/PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t) -> int | None:
    if t is None:
        return None
    return t.data_ptr()


def call(name: str, *args):
    """Invoke a status-returning entry point; raise with the library's message on failure."""
    global launch_count
    lib = load()
    rc = getattr(lib, name)(*args)
    launch_count += 1
    if rc != 0:
        raise B200Error(f"{name} failed ({rc}): {lib.b200_last_error().decode(errors='replace')}")


def query(name: str, *args):
    return getattr(load(), name)(*args)


def require_cuda(t: torch.Tensor, what: str = "tensor"):
    if not t.is_cuda:
        raise B200Error(f"{what} must live on a CUDA device: the native path has no CPU fallback")
