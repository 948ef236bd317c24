"""ctypes binding of ``libssb200.so`` (the C ABI declared in ``include/ssb200.h``).

The product path has NO CPU fallback: if the shared library is missing or a
call fails, a ``RuntimeError`` is raised.  ``build_library()`` compiles it
in-tree with ``nvcc`` for sm_90a (cross-compiles without a GPU).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
LIB_PATH = os.environ.get("SSB200_LIB", os.path.join(_HERE, "libssb200.so"))   # override: A/B builds while tuning
SOURCES = [os.path.join(_HERE, "csrc", "ssb200.cu")]
HEADERS = [os.path.join(_HERE, "csrc", "fft16.cuh"), os.path.join(_HERE, "csrc", "conv64k.cuh"),
           os.path.join(ROOT, "include", "ssb200.h")]

NVCC_FLAGS = ["-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
              "-lineinfo", "-O3", "-std=c++17"]

SSB_FLAG_SILENT = 1
PAD_MODES = {"reflect": 0, "constant": 1}

# numpy mirror of ssb_conv_term / ssb_req (include/ssb200.h)
TERM_DTYPE = np.dtype([("rir_offset", "<i8"), ("x_offset", "<i8"), ("rir_taps", "<i4"),
                       ("x_nw", "<i4"), ("x_wofs", "<i4"), ("reserved", "<i4")], align=True)
REQ_DTYPE = np.dtype([("term", TERM_DTYPE, (2,)), ("out_samples", "<i4"), ("flags", "<u4")], align=True)
assert TERM_DTYPE.itemsize == 32 and REQ_DTYPE.itemsize == 72


class Plan(C.Structure):
    _fields_ = [("log2n", C.c_int32), ("block", C.c_int32), ("sr", C.c_int32), ("n_blocks", C.c_int32),
                ("max_parts", C.c_int32), ("n_terms", C.c_int32), ("h_elems_per_env", C.c_int64)]


class Conv2dLayer(C.Structure):
    """ssb_conv2d_layer (include/ssb200.h)."""
    _fields_ = [("d_weight", C.c_void_p), ("d_bias", C.c_void_p), ("out_channels", C.c_int32), ("kh", C.c_int32),
                ("kw", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32), ("relu", C.c_int32)]


class ConvStackInput(C.Structure):
    """ssb_conv_stack_input (include/ssb200.h)."""
    _fields_ = [("d_x", C.c_void_p), ("d_depth", C.c_void_p), ("d_labels", C.c_void_p), ("label_stride", C.c_int64),
                ("kind", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("channels", C.c_int32),
                ("n_depth", C.c_int32), ("n_labels", C.c_int32)]


CONV_INPUT_SPECTROGRAM, CONV_INPUT_VISUAL, CONV_INPUT_MAP = 0, 1, 2


class ResnetConv(C.Structure):
    """ssb_resnet_conv (include/ssb200.h)."""
    _fields_ = [("d_weight", C.c_void_p), ("d_gamma", C.c_void_p), ("d_beta", C.c_void_p), ("d_mean", C.c_void_p),
                ("d_var", C.c_void_p), ("eps", C.c_float), ("reserved", C.c_int32)]


class SmtCnnInput(C.Structure):
    """ssb_smt_cnn_input (include/ssb200.h)."""
    _fields_ = [("d_obs", C.c_void_p), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("scale", C.c_int32),
                ("resized_h", C.c_int32), ("resized_w", C.c_int32), ("crop_y", C.c_int32), ("crop_x", C.c_int32),
                ("convs", ResnetConv * 20), ("d_fc_weight", C.c_void_p), ("d_fc_bias", C.c_void_p),
                ("fc_in", C.c_int32), ("n_out", C.c_int32)]


class RolloutField(C.Structure):
    """ssb_rollout_field (include/ssb200.h)."""
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("row_bytes", C.c_int64), ("src_t_stride", C.c_int64),
                ("src_outer_stride", C.c_int64), ("T", C.c_int32), ("outer", C.c_int32), ("on_host", C.c_int32),
                ("reserved", C.c_int32)]


class RolloutMemory(C.Structure):
    """ssb_rollout_memory (include/ssb200.h)."""
    _fields_ = [("d_masks", C.c_void_p), ("not_done", C.c_void_p), ("d_em_masks_out", C.c_void_p),
                ("d_status", C.c_void_p), ("total", C.c_int32), ("capacity", C.c_int32), ("idx", C.c_int32),
                ("step", C.c_int32), ("not_done_on_host", C.c_int32), ("reserved", C.c_int32)]


class Linear(C.Structure):
    """ssb_linear (include/ssb200.h)."""
    _fields_ = [("d_weight", C.c_void_p), ("d_bias", C.c_void_p)]


class LayerNorm(C.Structure):
    """ssb_layer_norm (include/ssb200.h)."""
    _fields_ = [("d_gamma", C.c_void_p), ("d_beta", C.c_void_p), ("eps", C.c_float), ("reserved", C.c_int32)]


class MapGeometry(C.Structure):
    """ssb_map_geometry (include/ssb200.h)."""
    _fields_ = [(n, C.c_int32) for n in ("internal_size", "stride", "map_size", "action_size", "ego_size", "encoding",
                                         "acoustic", "n_slots")]


class FrameSensor(C.Structure):
    """ssb_frame_sensor (include/ssb200.h)."""
    _fields_ = [("d_bank", C.c_void_p), ("d_stage", C.c_void_p), ("d_dst", C.c_void_p), ("h_index", C.c_void_p),
                ("h_fill", C.c_void_p), ("row_elems", C.c_int64), ("bank_rows", C.c_int64), ("dst_stride", C.c_int64),
                ("n_fill", C.c_int32), ("dtype", C.c_int32)]


FRAME_MAX_SENSORS, FRAME_MAX_N = 4, 256
FRAME_DTYPES = {np.dtype(np.uint8): 0, np.dtype(np.float32): 1}       # SSB_FRAME_U8, SSB_FRAME_F32


SMT_LINEARS = ("pose", "fuse1", "fuse2", "enc_qkv", "enc_out", "enc_ff1", "enc_ff2")
SMT_ENC_NORMS = ("enc_norm1", "enc_norm2", "enc_norm")
SMT_DEC_LINEARS = ("dec_sa_qkv", "dec_sa_out", "dec_ca_qkv", "dec_ca_out", "dec_ff1", "dec_ff2")
SMT_DEC_NORMS = ("dec_norm1", "dec_norm2", "dec_norm3", "dec_norm")


class SmtParams(C.Structure):
    """ssb_smt_params (include/ssb200.h)."""
    _fields_ = ([("d_in", C.c_int32), ("pose_index", C.c_int32), ("d_model", C.c_int32), ("n_heads", C.c_int32),
                 ("pretraining", C.c_int32)] + [(n, Linear) for n in SMT_LINEARS] + [(n, LayerNorm) for n in SMT_ENC_NORMS]
                + [(n, Linear) for n in SMT_DEC_LINEARS] + [(n, LayerNorm) for n in SMT_DEC_NORMS])


EXPORTS = {
    # name: (restype, argtypes)
    "ssb_version": (C.c_int, []),
    "ssb_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "ssb_destroy": (None, [C.c_void_p]),
    "ssb_last_error": (C.c_char_p, [C.c_void_p]),
    "ssb_launch_count": (C.c_int64, [C.c_void_p]),
    "ssb_set_conv_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "ssb_set_streams": (C.c_int, [C.c_void_p, C.c_int]),
    "ssb_set_chunks": (C.c_int, [C.c_void_p, C.c_int]),
    "ssb_set_debug": (C.c_int, [C.c_void_p, C.c_int]),
    "ssb_set_kernel_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "ssb_get_kernel_timing": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "ssb_make_plan": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(Plan)]),
    "ssb_spec_cols": (C.c_int, [C.c_int]),
    "ssb_source_windows": (C.c_int, [C.c_void_p, C.POINTER(Plan), C.c_void_p, C.c_int, C.c_int64, C.c_int,
                                     C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ssb_convolve_batch": (C.c_int, [C.c_void_p, C.POINTER(Plan), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "ssb_crossfade_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                      C.c_void_p, C.c_void_p]),
    "ssb_spectrogram_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "ssb_render_batch": (C.c_int, [C.c_void_p, C.POINTER(Plan), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "ssb_render_batch_host": (C.c_int, [C.c_void_p, C.POINTER(Plan), C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "ssb_host_copy_bytes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "ssb_sh_decode_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "ssb_sh_decode_multi_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_intensity_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ssb_audio_conv1_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ssb_audio_encoder_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(Conv2dLayer),
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_audio_encoder_category_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                   C.POINTER(Conv2dLayer), C.c_void_p, C.c_int, C.c_int64, C.c_void_p,
                                                   C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_visual_encoder_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int, C.POINTER(Conv2dLayer), C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_map_encoder_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.POINTER(Conv2dLayer), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "ssb_gru_step_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "ssb_gru_seq_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "ssb_gru_seq_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 12),
    "ssb_gru_seq_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 15),
    "ssb_conv_stack_train_workspace_bytes": (C.c_int64, [C.c_int, C.POINTER(ConvStackInput), C.POINTER(Conv2dLayer),
                                                         C.c_int, C.c_int, C.c_int]),
    "ssb_conv_stack_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(ConvStackInput),
                                                     C.POINTER(Conv2dLayer), C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                     C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_conv_stack_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(ConvStackInput),
                                                      C.POINTER(Conv2dLayer), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]),
    "ssb_policy_head_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_policy_head_train_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "ssb_policy_head_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5
                                            + [C.c_int] + [C.c_void_p] * 8),
    "ssb_policy_head_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 3
                                             + [C.c_int] + [C.c_void_p] * 13),
    "ssb_rollout_insert_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(RolloutField), C.c_int,
                                           C.POINTER(RolloutMemory), C.c_void_p]),
    "ssb_rollout_returns_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                            C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_void_p]),
    "ssb_rollout_gather_batch": (C.c_int, [C.c_void_p, C.POINTER(RolloutField), C.c_int, C.c_int, C.c_void_p,
                                           C.c_int64, C.c_void_p]),
    "ssb_belief_update_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_double, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    "ssb_resnet18_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(ResnetConv),
                                     C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ssb_smt_resnet18_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                         C.c_int64, C.POINTER(ResnetConv), C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p]),
    "ssb_smt_resnet18_train_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ssb_smt_resnet18_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                       C.c_int, C.c_int64, C.POINTER(ResnetConv), C.c_void_p,
                                                       C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                       C.c_void_p]),
    "ssb_smt_resnet18_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                        C.c_int, C.c_int64, C.POINTER(ResnetConv), C.c_void_p, C.c_int,
                                                        C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
                                                        C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p,
                                                        C.c_void_p, C.c_void_p]),
    "ssb_resnet18_train_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "ssb_resnet18_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                   C.POINTER(ResnetConv), C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                   C.c_int, C.c_float, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p,
                                                   C.c_void_p]),
    "ssb_resnet18_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                    C.POINTER(ResnetConv), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                    C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
                                                    C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p,
                                                    C.c_void_p, C.c_void_p]),
    "ssb_smt_cnn_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(SmtCnnInput), C.c_void_p, C.c_void_p]),
    "ssb_smt_cnn_train_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.POINTER(SmtCnnInput)]),
    "ssb_smt_cnn_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(SmtCnnInput), C.c_void_p,
                                                  C.c_void_p, C.c_void_p]),
    "ssb_smt_cnn_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(SmtCnnInput), C.c_void_p,
                                                   C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]),
    "ssb_smt_scratch_bytes": (C.c_int64, [C.c_int, C.c_int, C.POINTER(SmtParams)]),
    "ssb_smt_state_encoder_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.POINTER(SmtParams), C.c_void_p, C.c_void_p, C.c_void_p]),
    "ssb_smt_train_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.POINTER(SmtParams)]),
    "ssb_smt_state_encoder_train_forward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                            C.c_void_p, C.c_void_p, C.POINTER(SmtParams), C.c_void_p,
                                                            C.c_void_p, C.c_void_p]),
    "ssb_smt_state_encoder_train_backward_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                             C.c_void_p, C.c_void_p, C.POINTER(SmtParams), C.c_void_p,
                                                             C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p,
                                                             C.c_void_p, C.c_void_p]),
    "ssb_logmel_frames": (C.c_int, [C.c_int]),
    "ssb_mel_filterbank": (C.c_int, [C.c_int, C.c_int, C.c_void_p]),
    "ssb_logmel_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p]),
    "ssb_map_update_batch": (C.c_int, [C.c_void_p, C.POINTER(MapGeometry), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_int64, C.c_void_p]),
    "ssb_map_update_device_intensity_batch": (C.c_int, [C.c_void_p, C.POINTER(MapGeometry), C.c_void_p, C.c_void_p,
                                                        C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                                        C.c_int64, C.c_void_p]),
    "ssb_map_observe_batch": (C.c_int, [C.c_void_p, C.POINTER(MapGeometry), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_int64, C.c_void_p]),
    "ssb_frame_gather_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(FrameSensor), C.c_int, C.c_void_p]),
    "ssb_pcm16_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "ssb_pcm16_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
}

_lib = None


def build_library(force=False, verbose=False):
    """Compile libssb200.so in-tree for sm_90a.  Returns the path."""
    deps = SOURCES + HEADERS
    if (not force and os.path.exists(LIB_PATH)
            and os.path.getmtime(LIB_PATH) >= max(os.path.getmtime(p) for p in deps)):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stdout + res.stderr)
    return LIB_PATH


def load_library():
    """dlopen libssb200.so and declare prototypes.  Fails loudly when missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the audio observation path)")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in EXPORTS.items():
        fn = getattr(lib, name)        # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


class Context:
    """Owns one ``ssb_ctx`` (one per process and device)."""

    def __init__(self, device_index=0):
        self.lib = load_library()
        handle = C.c_void_p()
        rc = self.lib.ssb_create(int(device_index), C.byref(handle))
        self.handle = handle
        if rc != 0:
            msg = self.lib.ssb_last_error(handle).decode() if handle else "allocation failed"
            if handle:
                self.lib.ssb_destroy(handle)
                self.handle = None
            raise RuntimeError(f"ssb_create(device={device_index}) failed ({rc}): {msg}")

    def check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.ssb_last_error(self.handle).decode()}")

    def make_plan(self, sr, max_taps, n_terms=1, log2n=0):
        plan = Plan()
        self.check(self.lib.ssb_make_plan(self.handle, sr, max_taps, n_terms, log2n, C.byref(plan)), "ssb_make_plan")
        return plan

    KERNEL_NAMES = ("fwd_rir_kernel", "mac_ifft_kernel", "spectrogram_kernel", "fwd_src_kernel", "mac_bins_kernel",
                    "conv64k_kernel")

    def set_kernel_timing(self, enable):
        self.check(self.lib.ssb_set_kernel_timing(self.handle, int(bool(enable))), "ssb_set_kernel_timing")

    def get_kernel_timing(self):
        """{kernel: (summed ms, launches)} since the last call (synchronises)."""
        ms = (C.c_double * len(self.KERNEL_NAMES))()
        cnt = (C.c_int64 * len(self.KERNEL_NAMES))()
        self.check(self.lib.ssb_get_kernel_timing(self.handle, ms, cnt), "ssb_get_kernel_timing")
        return {n: (ms[i], cnt[i]) for i, n in enumerate(self.KERNEL_NAMES)}

    @property
    def launch_count(self):
        return int(self.lib.ssb_launch_count(self.handle))

    def close(self):
        if getattr(self, "handle", None):
            self.lib.ssb_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
