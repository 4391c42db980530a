"""ctypes binding of ``libdotaclient_b200.so`` (the C-ABI in ``include/dotaclient_b200.h``).

There is NO fallback: if the library is missing or a call fails, a ``RuntimeError`` is raised.
The library is built in-tree by ``dotaclient_b200.build`` (``__graft_entry__.build()``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdotaclient_b200.so")

_c = ctypes
_vp, _i32, _i64, _f32, _f64, _sz = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_float, _c.c_double, _c.c_size_t
_ptr5 = _c.c_void_p * 5


class GatherDesc(_c.Structure):
    """``dc_gather_desc``: one tensor of a ``dc_gather_columns`` call."""
    _fields_ = [("src", _vp), ("dst", _vp), ("outer", _i64), ("src_cols", _i64), ("row_bytes", _i64)]

# name -> (restype, argtypes); must list every symbol include/dotaclient_b200.h declares.
SIGNATURES = {
    "dc_version": (_i32, []),
    "dc_last_error": (_c.c_char_p, []),
    "dc_device_info": (_i32, [_c.POINTER(_i32)] * 3),
    "dc_gae_scan": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _vp, _vp, _vp]),
    "dc_vtrace_scan": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _f64, _f64, _vp, _vp, _vp, _vp]),
    "dc_gae_scan_indexed": (_i32, [_vp, _i32, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _vp, _vp, _vp]),
    "dc_vtrace_scan_indexed": (_i32, [_vp, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _f64, _f64, _vp,
                                      _vp, _vp, _vp]),
    "dc_upgo_scan": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _f64, _vp, _vp, _vp]),
    "dc_upgo_scan_indexed": (_i32, [_vp, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _f64, _f64, _f64, _vp, _vp,
                                    _vp]),
    "dc_gae_scan_heads": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _f64, _vp, _vp, _vp]),
    "dc_gae_scan_heads_indexed": (_i32, [_vp, _i32, _vp, _i32, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _f64, _vp, _vp,
                                         _vp]),
    "dc_value_heads_loss": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dc_gather_columns": (_i32, [_c.POINTER(GatherDesc), _i32, _vp, _i64, _vp]),
    "dc_gather_columns_fill": (_i32, [_c.POINTER(GatherDesc), _i32, _vp, _i64, _vp]),
    "dc_refresh_states": (_i32, [_i32, _i32, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp]),
    "dc_rnn_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "dc_rnn_seq_fwd": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "dc_rnn_seq_bwd": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "dc_rnn_seq_fwd_reset": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "dc_rnn_seq_bwd_reset": (_i32, [_i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp,
                                    _vp]),
    "dc_gemm_tf32x3_supported": (_i32, [_i64, _i32, _i32]),
    "dc_gemm_tf32x3": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _i64, _i32, _i32, _i32, _vp]),
    "dc_gemm_wgrad_workspace_bytes": (_sz, [_i32, _i32]),
    "dc_gemm_wgrad_tf32x3": (_i32, [_vp, _i32, _vp, _i32, _i64, _i32, _i32, _vp, _i32, _vp, _i32, _vp, _vp]),
    "dc_gemm_tf32x3_rows": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "dc_gemm_wgrad_tf32x3_rows": (_i32, [_vp, _i32, _vp, _i32, _vp, _i64, _vp, _i32, _i32, _vp, _i32, _vp, _i32, _vp, _vp]),
    "dc_unit_basic_bwd_workspace_bytes": (_sz, []),
    "dc_env_fwd": (_i32, [_vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "dc_env_bwd_workspace_bytes": (_sz, []),
    "dc_env_bwd": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp]),
    "dc_unit_wgrad_routed": (_i32, [_vp, _vp, _i32, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp]),
    "dc_unit_dgrad_fused": (_i32, [_vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp]),
    "dc_unit_dgrad_fused_mask": (_i32, [_vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i32, _vp,
                                        _vp]),
    "dc_gemm_unit_max": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _i32, _vp]),
    "dc_unit_embed_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _i32, _vp]),
    "dc_unit_embed_fwd_mask": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _i32, _vp]),
    "dc_target_unit_q_fwd": (_i32, [_vp, _i32, _c.c_void_p * 6, _vp, _vp, _vp, _i64, _vp]),
    "dc_target_unit_q_bwd": (_i32, [_vp, _c.c_void_p * 6, _vp, _vp, _vp, _i32, _i64, _vp]),
    "dc_target_unit_q_fwd_rows": (_i32, [_vp, _i32, _c.c_void_p * 6, _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "dc_target_unit_q_bwd_rows": (_i32, [_vp, _c.c_void_p * 6, _vp, _vp, _vp, _i32, _i64, _vp, _vp, _vp]),
    "dc_target_rows_workspace_bytes": (_sz, [_i64]),
    "dc_target_rows": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dc_rows_zero_inactive": (_i32, [_vp, _i64, _vp, _i32, _i32, _vp]),
    "dc_ppo_loss_fwd_bwd": (_i32, [_ptr5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _ptr5, _vp, _vp,
                                   _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_strided": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _f32, _f32,
                                           _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_dev": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp,
                                       _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_masked": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                                          _vp, _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_joint": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                                         _vp, _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_kl": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                                      _vp, _i32, _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_teacher": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp,
                                           _vp, _i64, _vp, _vp, _i32, _ptr5, _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp,
                                           _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_dual_clip": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _vp, _vp, _vp, _i64,
                                             _vp, _vp, _i64, _vp, _vp, _vp, _i32, _ptr5, _c.c_int64 * 5, _vp, _i64, _vp,
                                             _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dc_ppo_loss_fwd_bwd_bc": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _ptr5, _vp, _vp, _vp, _i64, _vp, _vp, _i64, _vp, _ptr5,
                                      _c.c_int64 * 5, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dc_selected_logp_rows": (_i32, [_ptr5, _ptr5, _ptr5, _i64, _vp, _vp, _vp]),
    "dc_value_norm_stats": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "dc_value_denorm": (_i32, [_vp, _i64, _i64, _f64, _f64, _vp, _vp]),
    "dc_value_head_rescale": (_i32, [_vp, _i64, _vp, _f64, _f64, _f64, _f64, _vp]),
    "dc_selected_logp": (_i32, [_ptr5, _ptr5, _ptr5, _i64, _vp, _vp]),
    "dc_select_actions": (_i32, [_ptr5, _c.c_int64 * 5, _ptr5, _vp, _i64, _vp, _vp, _vp]),
    "dc_grad_flags": (_i32, [_vp, _i64, _vp, _i32, _vp, _vp]),
    "dc_grad_finish": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _f64, _f64, _f64, _f64, _f64, _vp, _vp,
                              _vp, _vp]),
    "dc_grad_finish_dev": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp, _f64, _f64, _f64, _vp, _vp, _vp,
                                  _vp]),
    "dc_grad_finish_kl": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp, _f64, _f64, _f64, _vp, _vp, _vp,
                                 _vp]),
}

PPO_WORKSPACE_BYTES = 512
FINISH_WORKSPACE_BYTES = 1024
LOSS_SLOTS = 16
# the device hyper-parameter block of the `_dev` entry points (fp64, DC_HP_* in include/dotaclient_b200.h)
HPARAM_SLOTS = 10
HP_LR, HP_E_CLIP, HP_ENTROPY_COEF, HP_VF_COEF, HP_MAX_GRAD_NORM, HP_VALUE_CLIP = range(6)
HP_VALUE_NORM_MEAN, HP_VALUE_NORM_STD = 6, 7       # value normalisation (mu, sigma); sigma 0 = off
HP_KL_COEF, HP_KL_STOP = 8, 9                      # KL control: penalty beta, early-stop limit (0 = none)
# the PPO diagnostics written by dc_ppo_loss_fwd_bwd_dev (DC_STAT_* in include/dotaclient_b200.h)
PPO_STATS_SLOTS = 24
STAT_APPROX_KL, STAT_CLIP_FRACTION, STAT_EXPLAINED_VAR = 0, 6, 12
STAT_JOINT_APPROX_KL, STAT_JOINT_CLIP_FRACTION = 13, 14     # dc_ppo_loss_fwd_bwd_joint only
STAT_KL, STAT_KL_PENALTY = 16, 22                           # dc_ppo_loss_fwd_bwd_kl only (17..21: KL per head)
KL_ROW_FLOATS = 65          # entries of one token's masked log-prob row over the five heads (DC_KL_ROW_FLOATS)
# dc_ppo_loss_fwd_bwd_teacher's teacher_stats: 0 the KL to the teacher, 1..5 per head, 6 lambda * KL (DC_TEACHER_STATS_SLOTS)
TEACHER_STATS_SLOTS = 7
# dc_ppo_loss_fwd_bwd_bc's bc_stats: 0 the NLL, 1..5 per head, 6 the token accuracy, 7..11 per head (DC_BC_STATS_SLOTS)
BC_STATS_SLOTS = 12
# dc_ppo_loss_fwd_bwd_dual_clip's dual_clip_stats: 0 the mean bound fraction over the heads, 1..5 per head, 6 the joint
# ratio's (DC_DUAL_CLIP_STATS_SLOTS)
DUAL_CLIP_STATS_SLOTS = 7
FINISH_KL_METRICS = 6       # metrics of dc_grad_finish_kl: the four of dc_grad_finish, the all-ranks KL, the skip flag
VTRACE_STATS_SLOTS = 8      # per-segment fp64 sums written by dc_vtrace_scan (DC_VTRACE_STATS_SLOTS)
UPGO_STATS_SLOTS = 3        # per-segment fp64 sums written by dc_upgo_scan (DC_UPGO_STATS_SLOTS)
VALUE_HEADS_MAX = 10        # value heads of dc_gae_scan_heads / dc_value_heads_loss (DC_VALUE_HEADS_MAX)
VALUE_HEADS_STATS_SLOTS = 20    # dc_value_heads_loss: [k] value loss, [VALUE_HEADS_MAX + k] explained variance of head k
VALUE_HEADS_WORKSPACE_BYTES = 131072
GATHER_MAX_TENSORS = 32     # descriptors per dc_gather_columns call (DC_GATHER_MAX_TENSORS)
REFRESH_MAX_LAYERS = 16     # recurrent layers dc_refresh_states handles (DC_REFRESH_MAX_LAYERS)
MAX_PARAM_TENSORS = 96      # kMaxSeg of csrc/grad_finish.cu: parameter tensors dc_grad_flags / dc_grad_finish can handle

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def load():
    """Loads the shared library (once).  Raises if it has not been built -- no silent fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: build it with `python -m dotaclient_b200.build` (needs nvcc, sm_90a). "
            "dotaclient_b200 has no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def exported(name):
    lib = load()
    return hasattr(lib, name)


def check(rc, what):
    if rc != 0:
        msg = load().dc_last_error()
        raise RuntimeError("%s failed (code %d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def ptr5(tensors):
    return _ptr5(*[t.data_ptr() if t is not None else None for t in tensors])


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream
