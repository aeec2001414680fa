"""ctypes binding of libhebo_b200.so (the C ABI of include/hebo_b200.h).

The product path has no CPU / torch fallback: if the CUDA library is missing the import of the model
classes still works (so that host-only logic can be tested) but every compute call raises loudly.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libhebo_b200.so")

HB_OK, HB_ERR_INVALID, HB_ERR_NOT_PD, HB_ERR_CUDA = 0, 1, 2, 3
KERNEL_IDS = {"matern32": 0, "matern52": 1, "rbf": 2, "matern12": 4}   # HB_KERN_* of include/hebo_b200.h
HB_ACQ1_LCB, HB_ACQ1_MEAN, HB_ACQ1_SIGMA, HB_ACQ1_ABS_ETA = 0, 1, 2, 3   # hb_acq1_epilogue modes
HB_MAX_FEATURES = 4096   # d + sum(emb_sizes) a model may have (include/hebo_b200.h)
HB_MAX_OUTPUTS = 32      # outputs one batched fit trains together (hb_fit_multi_ex)
HB_MAX_OBJ = 8           # objectives of hb_nsga2_survive_k / hb_pareto_front_k
# deep-ensemble envelope (HB_DE_MAX_* of include/hebo_b200.h)
HB_DE_MAX_LAYERS, HB_DE_MAX_HIDDEN, HB_DE_MAX_OUT, HB_DE_MAX_IN, HB_DE_MAX_MEMBERS = 3, 256, 8, 256, 32
HB_DE_MAX_BATCH_FLOATS = 56000
HB_DE_EMBEDDING, HB_DE_ONEHOT = 0, 1
HB_FE_STG, HB_FE_CONCRETE, HB_FE_HARD_CONCRETE = 0, 1, 2
# random-forest envelope (HB_RF_MAX_* of include/hebo_b200.h)
HB_RF_MAX_ROWS, HB_RF_MAX_WIDTH, HB_RF_MAX_TREES = 8192, 4096, 1024
HB_RF_NAN_LEFT = 1 << 30   # flag of an internal node's feature word: NaN inputs go left (sklearn's missing_go_to_left)


class HeboB200Error(RuntimeError):
    pass


class NotPositiveDefinite(HeboB200Error):
    pass


class FitState(C.Structure):      # hb_fit_state_t
    _fields_ = [("hyp", C.c_void_p), ("L", C.c_void_p), ("Linv", C.c_void_p), ("alpha", C.c_void_p),
                ("Zt", C.c_void_p), ("scal", C.c_void_p), ("Linv_hi", C.c_void_p), ("Linv_lo", C.c_void_p),
                ("tab_s", C.c_void_p), ("emb_meta", C.c_void_p), ("grad", C.c_void_p), ("loss", C.c_void_p)]


class ModelSpec(C.Structure):     # hb_model_spec_t
    _fields_ = [("ard_kernel", C.c_int32), ("num_enum", C.c_int32), ("num_uniqs", C.POINTER(C.c_int32)),
                ("emb_sizes", C.POINTER(C.c_int32)), ("warp", C.c_int32)]


class DeSpec(C.Structure):        # hb_de_spec_t
    _fields_ = [("num_cont", C.c_int32), ("num_enum", C.c_int32), ("num_uniqs", C.POINTER(C.c_int32)),
                ("enum_trans", C.c_int32), ("num_layers", C.c_int32), ("num_hiddens", C.c_int32), ("num_out", C.c_int32),
                ("output_noise", C.c_int32), ("rand_prior", C.c_int32), ("noise_lb", C.c_float)]


class FeGate(C.Structure):        # hb_fe_gate_t
    _fields_ = [("kind", C.c_int32), ("temperature", C.c_float), ("start_temp", C.c_double), ("end_temp", C.c_double),
                ("anneal_base", C.c_double), ("mask_reg", C.c_float)]


class RfSpec(C.Structure):        # hb_rf_spec_t
    _fields_ = [("num_cont", C.c_int32), ("num_enum", C.c_int32), ("num_uniqs", C.POINTER(C.c_int32))]


_vp, _i64, _i32, _f32, _u64 = C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_uint64
_sp = C.POINTER(ModelSpec)
_dsp = C.POINTER(DeSpec)
_rsp = C.POINTER(RfSpec)
_fgp = C.POINTER(FeGate)

# name -> (restype, argtypes); must list every function declared in include/hebo_b200.h
SIGNATURES = {
    "hb_version": (_i32, []),
    "hb_last_error": (C.c_char_p, []),
    "hb_padded_n": (_i64, [_i64]),
    "hb_launch_count": (_i64, [_i32]),
    "hb_profile_enable": (_i32, [_i32]),
    "hb_profile_collect": (_i32, [C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
    "hb_vnorm_operand_kind": (_i32, []),
    "hb_num_params": (_i64, [_i64, _sp]),
    "hb_guard_stats": (_i32, [C.POINTER(C.c_uint64), _i32]),
    "hb_fit_workspace_bytes": (_i64, [_i64, _i64]),
    "hb_fit_workspace_bytes_ex": (_i64, [_i64, _i64, _sp]),
    "hb_posterior_workspace_bytes": (_i64, [_i64, _i64, _i64]),
    "hb_pareto_workspace_bytes": (_i64, [_i64]),
    "hb_transform_hypers": (_i32, [_vp, _i64, _f32, _vp, _vp]),
    "hb_median_pdist": (_i32, [_vp, _i64, _i64, _vp, _i64, _f32, _vp, _vp]),
    "hb_gram": (_i32, [_vp, _i64, _i64, _vp, _i32, _vp, _f32, _vp, _vp]),
    "hb_cholesky": (_i32, [_vp, _i64, _vp, _vp, _vp]),
    "hb_tri_inverse": (_i32, [_vp, _i64, _vp, _vp, _vp]),
    "hb_kinv": (_i32, [_vp, _i64, _vp, _vp]),
    "hb_tc_workspace_bytes": (_i64, [_i64]),
    "hb_cholesky_tc": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "hb_tri_inverse_tc": (_i32, [_vp, _i64, _vp, _vp, _i64, _vp]),
    "hb_kinv_tc": (_i32, [_i64, _vp, _vp, _i64, _vp]),
    "hb_solve_logdet": (_i32, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "hb_mll_grad": (_i32, [_vp, _i64, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp]),
    "hb_psgld_step": (_i32, [_vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _vp, _vp]),
    "hb_fit": (_i32, [_vp, _vp, _i64, _i64, _vp, _i32, _vp, _f32, _f32, _f32, _i32, _vp,
                      C.POINTER(C.c_float), _vp, _i64, _vp]),
    "hb_factorize": (_i32, [_vp, _vp, _i64, _i64, _vp, _i32, _vp, _f32, C.POINTER(C.c_float), _vp, _i64, _vp]),
    "hb_fit_state": (_i32, [_vp, _i64, _i64, C.POINTER(FitState)]),
    "hb_fit_state_ex": (_i32, [_vp, _i64, _i64, _sp, C.POINTER(FitState)]),
    "hb_fit_ex": (_i32, [_vp, _vp, _vp, _i64, _i64, _sp, _vp, _i32, _vp, _f32, _f32, _f32, _i32, _vp,
                         C.POINTER(C.c_float), _vp, _i64, _vp]),
    "hb_fit_multi_workspace_bytes": (_i64, [_i64, _i64, _sp, _i64]),
    "hb_fit_multi_ex": (_i32, [_vp, _vp, _vp, _i64, _i64, _sp, _i64, _vp, _i32, _vp, _f32, _f32, _f32, _i32, _vp,
                               C.POINTER(C.c_float), C.POINTER(C.c_int32), _vp, _i64, _vp]),
    "hb_factorize_ex": (_i32, [_vp, _vp, _vp, _i64, _i64, _sp, _vp, _i32, _vp, _f32, C.POINTER(C.c_float), _vp, _i64, _vp]),
    "hb_mll_fwd_bwd": (_i32, [_vp, _vp, _vp, _i64, _i64, _sp, _vp, _i32, _vp, _f32, _f32, _f32, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_posterior_mace_ex": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _sp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32,
                                    _f32, _f32, _i32, _f32, _f32, _f32, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "hb_posterior_grad_ex": (_i32, [_vp, _vp, _i64, _i64, _i64, _sp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32,
                                    _i32, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "hb_posterior_mace": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32, _i32,
                                 _f32, _f32, _f32, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "hb_posterior_grad": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32, _i32,
                                 _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "hb_sample_workspace_bytes": (_i64, [_i64, _i64, _sp, _i64]),
    "hb_sample_y": (_i32, [_vp, _vp, _i64, _i64, _i64, _sp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32, _i32, _vp, _i32,
                           _vp, C.POINTER(C.c_float), _vp, _i64, _vp]),
    "hb_sample_y_batch": (_i32, [_vp, _vp, _i64, _i64, _i64, _sp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32, _i32, _vp,
                                 _u64, _u64, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_mace_epilogue": (_i32, [_vp, _vp, _i64, _f32, _f32, _f32, _f32, _vp, _vp, _u64, _vp, _vp]),
    "hb_acq1_epilogue": (_i32, [_vp, _vp, _i64, _i32, _f32, _f32, _vp, _vp]),
    "hb_general_acq_epilogue": (_i32, [_vp, _vp, _i64, _i64, _i64, _f32, _f32, _vp, _vp, _u64, _u64, _vp, _vp, _vp, _vp]),
    "hb_mo_lcb_epilogue": (_i32, [_vp, _vp, _i64, _f32, _f32, _f32, _vp, _u64, _u64, _vp, _vp, _vp]),
    "hb_pareto_front3": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "hb_pareto_front_k": (_i32, [_vp, _i64, _i64, _vp, _vp, _vp, _i64, _vp]),
    "hb_nsga2_init": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _u64, _vp, _vp, _vp]),
    "hb_nsga2_mate": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _u64, _i32, _vp, _vp, _vp, _vp]),
    "hb_nsga2_survive": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "hb_nsga2_workspace_bytes": (_i64, [_i64, _i64]),
    "hb_nsga2_survive_ex": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_nsga2_survive_cv": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_ga_survive": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_ga_survive_cv": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_nsga2_workspace_bytes_k": (_i64, [_i64, _i64, _i64]),
    "hb_nsga2_survive_k": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "hb_embed_violation_workspace_bytes":(_i64, [_i64, _i64, _i64]),
    "hb_embed_violation": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _vp]),
    "hb_front_merge_workspace_bytes": (_i64, [_i64, _i64]),
    "hb_front_pack": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "hb_front_merge": (_i32, [_vp, _i64, _i64, _vp, _vp, _i64, _vp]),
    "hb_de_num_params": (_i64, [_dsp]),
    "hb_de_fit_workspace_bytes": (_i64, [_dsp, _i64]),
    "hb_de_fit": (_i32, [_vp, _vp, _vp, _i64, _dsp, _i64, _vp, C.c_double, _f32, _i64, _i64, _vp, _u64, _vp, _vp, _i64, _vp]),
    "hb_de_predict": (_i32, [_vp, _vp, _i64, _dsp, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "hb_de_predict_grad": (_i32, [_vp, _vp, _i64, _dsp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "hb_de_fit_batch": (_i32, [_vp, _vp, _vp, C.POINTER(C.c_int64), _i64, _dsp, _i64, _vp, C.c_double, _f32, _i64, _i64,
                               C.POINTER(C.c_uint64), _vp, _vp, _i64, _vp]),
    "hb_de_predict_batch": (_i32, [_vp, _vp, _i64, _dsp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _u64, _u64,
                                   _vp, _vp]),
    "hb_fe_num_params": (_i64, [_dsp]),
    "hb_fe_fit_workspace_bytes": (_i64, [_dsp, _i64]),
    "hb_fe_fit": (_i32, [_vp, _vp, _vp, _i64, _dsp, _fgp, _i64, _vp, C.c_double, _f32, _i64, _i64, _vp, _vp, _u64, _vp, _vp,
                         _i64, _vp]),
    "hb_fe_predict": (_i32, [_vp, _vp, _i64, _dsp, _fgp, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _u64, _u64, _vp, _vp, _vp]),
    "hb_gumbel_num_params": (_i64, [_dsp, _i64]),
    "hb_gumbel_fit_workspace_bytes": (_i64, [_dsp, _i64, _i64]),
    "hb_gumbel_fit": (_i32, [_vp, _vp, _vp, _i64, _dsp, _i64, _i64, _vp, C.c_double, _f32, _i64, _i64, _vp, _vp, _u64, _vp,
                             _vp, _i64, _vp]),
    "hb_gumbel_predict": (_i32, [_vp, _vp, _i64, _dsp, _i64, _f32, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _u64, _u64, _vp,
                                 _vp, _vp, _i64, _vp]),
    "hb_rf_fit_workspace_bytes": (_i64, [_i64, _rsp, _i64, _i64]),
    "hb_rf_forest_bytes": (_i64, [_rsp, _i64, _i64, _i64]),
    "hb_rf_fit": (_i32, [_vp, _vp, _vp, _i64, _rsp, _i64, _i64, _vp, _u64, _vp, _vp, _vp, _i64, _vp]),
    "hb_rf_predict": (_i32, [_vp, _vp, _i64, _rsp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _u64, _u64, _vp, _vp]),
    "hb_rf_load": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _rsp, _i64, _i64, _vp, _vp]),
    "hb_ehvi_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64]),
    "hb_ehvi": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _vp]),
}

_lib = None


def available() -> bool:
    return os.path.isfile(LIB_PATH)


def lib():
    """Load (once) and return the bound library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not available():
            raise HeboB200Error(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  hebo_b200 has no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status: int, what: str) -> None:
    if status == HB_OK:
        return
    if status == HB_ERR_NOT_PD:
        raise NotPositiveDefinite(f"{what}: matrix not positive definite (jitter ladder exhausted)")
    if status == HB_ERR_CUDA:
        raise HeboB200Error(f"{what}: CUDA error: {lib().hb_last_error().decode()}")
    raise HeboB200Error(f"{what}: invalid argument (status {status})")


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
