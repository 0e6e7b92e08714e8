"""ctypes binding of libzaremba_b200.so (the C ABI in include/zaremba_b200.h).

There is no CPU implementation behind this module: if the shared library is missing it is
built with nvcc, and if it cannot be built or there is no CUDA device the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

MAX_LAYERS = 8
MAX_BEAMS = 32
MAX_EXPERTS = 32
ENGINE_SIMT = 0
ENGINE_TC = 1
TIED_EMBEDDING = 1   # zrb_config.flags bit ZRB_TIED_EMBEDDING

_f32p = C.POINTER(C.c_float)
_vp = C.c_void_p


class ZrbConfig(C.Structure):
    _fields_ = [("vocab", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32),
                ("max_seq", C.c_int32), ("max_batch", C.c_int32), ("engine", C.c_int32),
                ("dropout", C.c_float), ("flags", C.c_int32)]


class ZrbParams(C.Structure):
    _fields_ = [("embed_w", _vp),
                ("w_ih", _vp * MAX_LAYERS), ("w_hh", _vp * MAX_LAYERS),
                ("b_ih", _vp * MAX_LAYERS), ("b_hh", _vp * MAX_LAYERS),
                ("fc_w", _vp), ("fc_b", _vp)]


class ZrbMosParams(ZrbParams):
    """zrb_mos_params: a ZrbParams (its `base`) followed by the Mixture-of-Softmaxes head; passes wherever a
    POINTER(ZrbParams) is expected"""
    _fields_ = [("prior_w", _vp), ("latent_w", _vp), ("latent_b", _vp)]


class ZrbStates(C.Structure):
    _fields_ = [("h", _vp * MAX_LAYERS), ("c", _vp * MAX_LAYERS)]


class ZrbSampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("reserved", C.c_int32),
                ("seed", C.c_uint64)]


class ZrbError(RuntimeError):
    pass


_SIGNATURES = {
    "zrb_last_error": (C.c_char_p, []),
    "zrb_version": (C.c_char_p, []),
    "zrb_launch_count": (C.c_int64, []),
    "zrb_ctx_create": (C.c_int, [C.POINTER(ZrbConfig), C.POINTER(_vp)]),
    "zrb_ctx_create_widths": (C.c_int, [C.POINTER(ZrbConfig), C.POINTER(C.c_int32), C.POINTER(_vp)]),
    "zrb_ctx_create_mos": (C.c_int, [C.POINTER(ZrbConfig), C.POINTER(C.c_int32), C.c_int32, C.POINTER(_vp)]),
    "zrb_set_mos_dropout": (C.c_int, [_vp, C.c_float]),
    "zrb_set_zoneout": (C.c_int, [_vp, C.c_float, C.c_float]),
    "zrb_ctx_destroy": (None, [_vp]),
    "zrb_ctx_workspace_bytes": (C.c_int64, [_vp]),
    "zrb_params_changed": (C.c_int, [_vp]),
    "zrb_dropout_mask": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int32, C.c_int64, C.c_float, _vp, _vp]),
    "zrb_set_explicit_masks": (C.c_int, [_vp, C.POINTER(_vp)]),
    "zrb_set_variational_dropout": (C.c_int, [_vp, C.c_int32, C.c_float]),
    "zrb_set_weight_drop": (C.c_int, [_vp, C.c_float, C.c_uint64]),
    "zrb_set_embed_dropout": (C.c_int, [_vp, C.c_float, C.c_uint64]),
    "zrb_set_activation_reg": (C.c_int, [_vp, C.c_float, C.c_float]),
    "zrb_activation_reg": (C.c_int, [_vp, _vp, _vp]),
    "zrb_forward": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                              C.POINTER(ZrbStates), _vp, C.c_int32, C.c_uint64, C.c_uint64, _vp]),
    "zrb_backward": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, C.POINTER(ZrbParams), _vp]),
    "zrb_softmax_nll": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp, _vp, _vp]),
    "zrb_clip_sgd": (C.c_int, [_vp, C.c_int32, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(C.c_int64),
                               C.c_float, C.c_float, _vp, _vp]),
    "zrb_train_step_grads": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), _vp, _vp, C.c_int32,
                                       C.c_int32, C.POINTER(ZrbStates), C.POINTER(ZrbStates), C.c_uint64,
                                       C.c_uint64, _vp, _vp]),
    "zrb_train_step_begin": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), _vp, _vp, C.c_int32,
                                       C.c_int32, C.POINTER(ZrbStates), C.POINTER(ZrbStates), C.c_uint64,
                                       C.c_uint64, _vp, _vp]),
    "zrb_train_step_layer": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), C.c_int32, _vp]),
    "zrb_set_embed_sparse": (C.c_int, [_vp, C.c_int32]),
    "zrb_set_keep_clipped_grads": (C.c_int, [_vp, C.c_int32]),
    "zrb_set_embed_rows_out": (C.c_int, [_vp, _vp]),
    "zrb_embed_scatter_rows": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int64, _vp]),
    "zrb_train_step_update": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), C.c_float, C.c_float,
                                        _vp, _vp]),
    "zrb_eval_step": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                                C.POINTER(ZrbStates), _vp, _vp, _vp]),
    "zrb_sample": (C.c_int, [_vp, C.c_int64, C.c_int32, C.c_int32, C.POINTER(ZrbSampling), C.c_uint64, _vp, _vp, _vp]),
    "zrb_generate": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                               C.POINTER(ZrbStates), C.c_int32, C.POINTER(ZrbSampling), C.c_uint64, _vp, _vp, _vp]),
    "zrb_beam_step": (C.c_int, [_vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, C.c_int32, _vp,
                                _vp, _vp, _vp, _vp]),
    "zrb_beam_search": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                                  C.POINTER(ZrbStates), C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp, _vp]),
    "zrb_cache_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_vp)]),
    "zrb_cache_reset": (C.c_int, [_vp]),
    "zrb_cache_destroy": (None, [_vp]),
    "zrb_cache_step": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, C.c_float, _vp, _vp]),
    "zrb_eval_step_cache": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp, _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                                      C.POINTER(ZrbStates), _vp, C.c_float, C.c_float, _vp, _vp, _vp, _vp]),
    "zrb_grad_stats_step": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), C.POINTER(ZrbParams), _vp, _vp,
                                      C.c_int32, C.c_int32, C.POINTER(ZrbStates), C.POINTER(ZrbStates), _vp, _vp]),
    "zrb_grad_stats_finish": (C.c_int, [_vp, C.POINTER(ZrbParams), C.c_int64, _vp, _vp]),
    "zrb_dyneval_step": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), C.POINTER(ZrbParams),
                                   C.POINTER(ZrbParams), _vp, _vp, _vp, C.c_int32, C.c_int32, C.POINTER(ZrbStates),
                                   C.POINTER(ZrbStates), C.c_float, C.c_float, C.c_float, _vp, _vp]),
    "zrb_train_step_host": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), _vp, _vp, C.c_int32,
                                      C.c_int32, C.POINTER(ZrbStates), C.POINTER(ZrbStates), C.c_uint64,
                                      C.c_uint64, C.c_float, C.c_float, _vp, _vp, _vp]),
    "zrb_set_lazy_update": (C.c_int, [_vp, C.c_int32]),
    "zrb_flush_updates": (C.c_int, [_vp, _vp]),
    "zrb_set_average": (C.c_int, [_vp, C.POINTER(ZrbParams)]),
    "zrb_average_count": (C.c_int, [_vp, C.POINTER(C.c_int64)]),
    "zrb_swap_average": (C.c_int, [_vp, C.POINTER(ZrbParams), _vp]),
    "zrb_set_adam": (C.c_int, [_vp, C.POINTER(ZrbParams), C.POINTER(ZrbParams), C.c_float, C.c_float, C.c_float,
                               C.c_int64]),
    "zrb_check_health": (C.c_int, [_vp]),
    "zrb_rec_plans": (C.c_int, [_vp, _vp]),
    "zrb_rec_plans_layer": (C.c_int, [_vp, C.c_int32, _vp]),
    "zrb_dp_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int64, C.POINTER(_vp)]),
    "zrb_dp_destroy": (None, [_vp]),
    "zrb_dp_grad_buffer": (_vp, [_vp]),
    "zrb_dp_export": (C.c_int, [_vp, _vp]),
    "zrb_dp_import": (C.c_int, [_vp, _vp]),
    "zrb_dp_begin_step": (C.c_int, [_vp, _vp]),
    "zrb_dp_finish_step": (C.c_int, [_vp, _vp]),
    "zrb_dp_allreduce_bucket": (C.c_int, [_vp, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _vp]),
    "zrb_lstm_layer_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "zrb_lstm_layer_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "zrb_prof_enable": (C.c_int, [_vp, C.c_int32]),
    "zrb_prof_read": (C.c_int, [_vp, _vp, _vp]),
    "zrb_prof_rec_trace": (C.c_int, [_vp, _vp, C.c_int32]),
    "zrb_gemm_f32": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                               C.c_float, _vp]),
    "zrb_gemm_f16": (C.c_int, [_vp, C.c_int64, C.c_int32, _vp, C.c_int64, C.c_int32, _vp, C.c_int64, C.c_int32,
                               C.c_int32, C.c_int32, C.c_float, _vp, C.c_int32, _vp]),
}

PROF_CLASSES = ["embed_fwd", "gemm_in", "rec_fwd", "proj_fwd", "softmax", "proj_bwd", "rec_bwd", "gemm_dx",
                "gemm_wgrad", "embed_bwd", "clip_sgd", "pack"]
REC_PLAN_FIELDS = ["ok", "KS", "U", "G", "nCTA", "GBi", "Kc", "KcS"]

_lib = None


def exported_symbols():
    """Names include/zaremba_b200.h declares (kept in step with the header by a test)."""
    return sorted(_SIGNATURES)


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if build_if_missing and _build.needs_build():
        _build.build()
    if not os.path.exists(path):
        raise ZrbError(f"{path} is missing and could not be built: zaremba_b200 has no CPU fallback")
    lib = C.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise ZrbError(f"libzaremba_b200 error {rc}: {load().zrb_last_error().decode()}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def rec_plans(ctx, layer=None):
    """zrb_rec_plans (layer None) or zrb_rec_plans_layer: {"fwd": {field: value}, "bwd": {...}} for a tensor-core
    context (fields: REC_PLAN_FIELDS)."""
    out = (C.c_int32 * 16)()
    if layer is None:
        check(load().zrb_rec_plans(ctx, out))
    else:
        check(load().zrb_rec_plans_layer(ctx, int(layer), out))
    return {d: dict(zip(REC_PLAN_FIELDS, out[8 * i:8 * i + 8])) for i, d in enumerate(("fwd", "bwd"))}
