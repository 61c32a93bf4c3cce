"""ctypes binding of libparakeet_b200.so (the C-ABI declared in include/parakeet_b200.h).

The product path has no CPU fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libparakeet_b200.so")

PK_ACT_NONE, PK_ACT_RELU, PK_ACT_TANH = 0, 1, 2


class PkError(RuntimeError):
    pass


class Operand(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("batch_stride", C.c_int64), ("ld", C.c_int32),
                ("rows", C.c_int32), ("cols", C.c_int32), ("batches", C.c_int32), ("bmul", C.c_int32),
                ("hmul", C.c_int32), ("col0", C.c_int32), ("colh", C.c_int32)]


class ConvGemmArgs(C.Structure):
    _fields_ = [("a", Operand), ("b", Operand), ("batch", C.c_int32), ("heads", C.c_int32), ("m", C.c_int32),
                ("n", C.c_int32), ("k", C.c_int32), ("taps", C.c_int32), ("dil", C.c_int32), ("pad", C.c_int32),
                ("scale", C.c_float), ("bias", C.c_void_p), ("act", C.c_int32), ("residual", C.c_void_p),
                ("lens", C.c_void_p), ("y_f32", C.c_void_p), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p),
                ("y_batch_stride", C.c_int64), ("y_head_stride", C.c_int64), ("y_ld", C.c_int32),
                ("passes", C.c_int32)]


class GemmEpilogue(C.Structure):
    _fields_ = [("mode", C.c_int32), ("channels", C.c_int32), ("residual", C.c_void_p), ("residual_batch_stride", C.c_int64),
                ("residual_ld", C.c_int32), ("skip_init", C.c_int32), ("state", C.c_void_p), ("skip", C.c_void_p),
                ("buf_hi", C.c_void_p), ("buf_lo", C.c_void_p), ("buf_ld", C.c_int32), ("buf_col0", C.c_int32)]


PK_EPI_NONE, PK_EPI_GATE, PK_EPI_WF_UPDATE = 0, 1, 2

_lib = None


def lib():
    """Load (once) and return the ctypes handle; raises PkError when the CUDA library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PkError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.pk_version.restype = C.c_int
        L.pk_last_error.restype = C.c_char_p
        L.pk_launch_count.restype = C.c_int64
        _declare(L)
        _lib = L
    return _lib


class PwgLayerArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("t", C.c_int32), ("dilation", C.c_int32), ("aux_channels", C.c_int32),
                ("lens", C.c_void_p), ("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("y_hi", C.c_void_p),
                ("y_lo", C.c_void_p), ("c_hi", C.c_void_p), ("c_lo", C.c_void_p), ("w1_hi", C.c_void_p),
                ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p), ("bias1", C.c_void_p),
                ("bias2", C.c_void_p), ("skip", C.c_void_p), ("skip_init", C.c_int32)]


class PwgLayerFcArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("t", C.c_int32), ("dilation", C.c_int32), ("hop", C.c_int32), ("lens", C.c_void_p),
                ("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("u_hi", C.c_void_p),
                ("u_lo", C.c_void_p), ("u_rows", C.c_int32), ("u_period", C.c_int32), ("u_start_row", C.c_int32),
                ("u_end_base", C.c_int32), ("p_rows", C.c_int32), ("p_ld", C.c_int32),
                ("p_frames", C.c_int32), ("p_row0", C.c_int32), ("p_hi", C.c_void_p), ("p_lo", C.c_void_p),
                ("w1_hi", C.c_void_p), ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p),
                ("bias1", C.c_void_p), ("bias2", C.c_void_p), ("skip", C.c_void_p), ("skip_init", C.c_int32)]


class WaveflowLayerArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_mels", C.c_int32),
                ("dilation", C.c_int32), ("slot", C.c_int32), ("buf_hi", C.c_void_p), ("buf_lo", C.c_void_p),
                ("cond_hi", C.c_void_p), ("cond_lo", C.c_void_p), ("cond_batch_stride", C.c_int64),
                ("w1_hi", C.c_void_p), ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p),
                ("bias1", C.c_void_p), ("bias2", C.c_void_p), ("next_hi", C.c_void_p), ("next_lo", C.c_void_p),
                ("skip", C.c_void_p), ("skip_init", C.c_int32)]


class WaveflowFlowArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_mels", C.c_int32),
                ("n_layers", C.c_int32), ("n_group", C.c_int32), ("cond_rows", C.c_void_p), ("ring_hi", C.c_void_p),
                ("ring_lo", C.c_void_p), ("cond_hi", C.c_void_p), ("cond_lo", C.c_void_p), ("w1_hi", C.c_void_p),
                ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p), ("bias1", C.c_void_p),
                ("bias2", C.c_void_p), ("in_w", C.c_void_p), ("in_b", C.c_void_p), ("out_w", C.c_void_p),
                ("out_b", C.c_void_p), ("z", C.c_void_p), ("x", C.c_void_p), ("skip", C.c_void_p), ("flags", C.c_void_p),
                ("flags_len", C.c_int64)]


class WaveflowForwardLayerArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_mels", C.c_int32),
                ("n_group", C.c_int32), ("dilation", C.c_int32), ("cond_rows", C.c_void_p), ("x_hi", C.c_void_p),
                ("x_lo", C.c_void_p), ("cond_hi", C.c_void_p), ("cond_lo", C.c_void_p), ("w1_hi", C.c_void_p),
                ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p), ("bias1", C.c_void_p),
                ("bias2", C.c_void_p), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("skip", C.c_void_p),
                ("skip_init", C.c_int32)]


class WaveflowForwardTailArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_group", C.c_int32),
                ("skip", C.c_void_p), ("out_w", C.c_void_p), ("out_b", C.c_void_p), ("x", C.c_void_p), ("perm", C.c_void_p),
                ("x_next", C.c_void_p), ("in_w", C.c_void_p), ("in_b", C.c_void_p), ("next_hi", C.c_void_p),
                ("next_lo", C.c_void_p), ("log_det", C.c_void_p), ("partials", C.c_void_p), ("counter", C.c_void_p)]


class WaveflowBackwardLayerArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_group", C.c_int32), ("dilation", C.c_int32),
                ("has_gemm1", C.c_int32), ("has_gemm2", C.c_int32), ("dh_ld", C.c_int32), ("dh_in_hi", C.c_void_p), ("dh_in_lo", C.c_void_p),
                ("w1_hi", C.c_void_p), ("w1_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p), ("dx", C.c_void_p),
                ("a2_hi", C.c_void_p), ("a2_lo", C.c_void_p), ("h", C.c_void_p), ("dh_out_hi", C.c_void_p), ("dh_out_lo", C.c_void_p)]


WAVEFLOW_TAIL_PARTIALS = 1024      # fp32 scratch elements pk_waveflow_forward_tail needs


class SsResidualBlockArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("t", C.c_int32), ("channels", C.c_int32), ("n_convs", C.c_int32), ("taps", C.c_int32),
                ("pad_left", C.c_int32), ("lens", C.c_void_p), ("x", C.c_void_p), ("x_hi", C.c_void_p), ("x_lo", C.c_void_p),
                ("w1_hi", C.c_void_p), ("w1_lo", C.c_void_p), ("bias1", C.c_void_p), ("scale1", C.c_void_p), ("shift1", C.c_void_p),
                ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p), ("bias2", C.c_void_p), ("scale2", C.c_void_p), ("shift2", C.c_void_p),
                ("y", C.c_void_p), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p)]


class Taco2DecodeArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("t_enc", C.c_int32), ("d_enc", C.c_int32), ("dmr", C.c_int32), ("steps", C.c_int32),
                ("teacher", C.c_int32), ("loc_k", C.c_int32), ("p_prenet", C.c_float), ("seed", C.c_uint64)] + \
        [(n, C.c_void_p) for n in ("keys", "pkeys", "text_lens", "mels", "pre_w1", "pre_w2", "att_w", "att_b_ih", "att_b_hh", "q_w",
                                   "loc_w", "v_w", "dec_w", "dec_b_ih", "dec_b_hh", "proj_w", "proj_b", "stop_w", "stop_b",
                                   "workspace")] + \
        [("workspace_len", C.c_int64)] + [(n, C.c_void_p) for n in ("mel_out", "align_out", "stop_out", "frames")] + \
        [("prof", C.c_void_p), ("prof_len", C.c_int64)]


class AttentionArgs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("q_hi", "q_lo", "k_hi", "k_lo", "vt_hi", "vt_lo")] + \
        [(n, C.c_int32) for n in ("batch", "t_q", "t_k", "heads", "dk", "tp", "q_ld", "k_ld", "q_col0", "k_col0", "causal")] + \
        [("key_lens", C.c_void_p), ("row_lens", C.c_void_p), ("scale", C.c_float), ("ctx_hi", C.c_void_p), ("ctx_lo", C.c_void_p)]


class TtsDecodeArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("t_enc", "adim", "heads", "units", "odim", "r", "prenet_layers", "prenet_units", "layers", "steps",
                                         "minlen", "maxlen")] + \
        [("threshold", C.c_float), ("p_prenet", C.c_float), ("seed", C.c_uint64)] + \
        [(n, C.c_void_p) for n in ("mem_kv", "pre_w", "pre_b", "in_w", "in_b", "pe", "layer_w", "norm", "out_w", "out_b", "workspace")] + \
        [("workspace_len", C.c_int64)] + [(n, C.c_void_p) for n in ("outs", "probs", "att_ws", "frames")]


def _declare(L):
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    sigs = {
        "pk_split_f32": [vp, vp, vp, i64, vp],
        "pk_conv_gemm": [C.POINTER(ConvGemmArgs), vp],
        "pk_conv_gemm_simt": [C.POINTER(ConvGemmArgs), vp],
        "pk_conv_gemm_ex": [C.POINTER(ConvGemmArgs), C.POINTER(GemmEpilogue), vp],
        "pk_length_regulator_lens": [vp, i32, i32, vp, vp],
        "pk_length_regulate": [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp],
        "pk_pwg_upsample": [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp],
        "pk_pwg_first_conv": [vp, vp, vp, vp, i32, i32, vp, vp, vp],
        "pk_pwg_residual_layer": [C.POINTER(PwgLayerArgs), vp],
        "pk_pwg_residual_layer_fc": [C.POINTER(PwgLayerFcArgs), vp],
        "pk_waveflow_layer": [C.POINTER(WaveflowLayerArgs), vp],
        "pk_waveflow_flow": [C.POINTER(WaveflowFlowArgs), vp],
        "pk_waveflow_forward_layer": [C.POINTER(WaveflowForwardLayerArgs), vp],
        "pk_waveflow_forward_tail": [C.POINTER(WaveflowForwardTailArgs), vp],
        "pk_waveflow_nll": [vp, vp, i64, f32, vp, vp],
        "pk_ss_residual_block": [C.POINTER(SsResidualBlockArgs), vp],
        "pk_ss_bn_train_fwd": [vp, i64, i32, vp, vp, f32, f32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp],
        "pk_ss_bn_relu_bwd": [vp, vp, vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp, vp],
        "pk_ss_loss": [vp, vp, vp, i32, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp],
        "pk_pwg_tail": [vp, vp, vp, vp, vp, vp, f32, i64, vp, vp],
        "pk_embed_pe": [vp, vp, i32, i32, vp, vp, vp, i32, i32, i32, vp, vp],
        "pk_layer_norm": [vp, vp, vp, f32, vp, i32, i32, i32, vp, vp, vp, vp],
        "pk_masked_softmax": [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp],
        "pk_transpose_heads": [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, vp],
        "pk_l2_normalize": [vp, i32, i32, i32, f32, vp, vp],
        "pk_fused_attention": [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, f32, vp, vp, vp],
        "pk_duration_post": [vp, vp, i32, i32, f32, vp, vp, vp],
        "pk_duration_scale": [vp, f32, i64, vp, vp],
        "pk_mask_rows": [vp, vp, i32, i32, i32, vp],
        "pk_variance_embed_add": [vp, vp, vp, vp, vp, i32, vp, vp, i32, vp, i32, i32, i32, vp, vp],
        "pk_zscore": [vp, vp, vp, i32, i64, i32, vp, vp],
        "pk_fs2_loss": [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp],
        "pk_transpose_planes": [vp, vp, i32, i32, i64, i32, i32, i32, i32, i32, vp, vp, i64, i64, vp],
        "pk_layer_norm_bwd": [vp, vp, vp, f32, i64, i32, vp, i32, vp, vp, vp],
        "pk_softmax_bwd": [vp, vp, vp, i64, i32, i32, f32, vp, vp, vp],
        "pk_colsum": [vp, i64, i32, vp, vp],
        "pk_sum_slices": [vp, i32, i64, vp, vp],
        "pk_colsum_split": [vp, vp, i64, i32, i32, vp, vp],
        "pk_batch_norm_train": [vp, i64, i32, vp, vp, f32, i32, f32, vp, vp, vp, vp, vp, vp, vp, vp, vp],
        "pk_batch_norm_bwd": [vp, vp, vp, vp, vp, vp, i32, i64, i32, vp, vp, vp],
        "pk_relu_bwd": [vp, vp, i64, vp, vp, vp, vp],
        "pk_axpy": [f32, vp, i64, vp, vp],
        "pk_fs2_loss_bwd": [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp],
        "pk_embed_pe_bwd": [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp],
        "pk_length_regulate_bwd": [vp, vp, i32, i32, i32, i32, vp, vp],
        "pk_scalar_conv_wgrad": [vp, vp, i32, i32, i32, i32, vp, vp, vp],
        "pk_adam": [vp, vp, vp, vp, i64, f32, f32, f32, f32, i32, f32, vp],
        "pk_spk_embed_fwd": [vp, i32, i32, vp, i32, i32, f32, vp, vp, vp],
        "pk_spk_time_sum": [vp, i32, i32, i32, i32, i32, vp, i32, vp, vp],
        "pk_spk_normalize_bwd": [vp, vp, vp, vp, i32, i32, i32, i32, f32, vp, vp],
        "pk_spk_table_grad": [vp, vp, i32, i32, i32, i32, vp, vp],
        "pk_gate_fwd": [vp, i64, i32, vp, vp, vp, vp],
        "pk_gate_bwd": [vp, vp, i64, i32, vp, vp],
        "pk_leaky_relu": [vp, i64, f32, vp, vp, vp, vp],
        "pk_leaky_relu_bwd": [vp, vp, i64, f32, vp, vp],
        "pk_weight_norm_fwd": [vp, vp, i32, i32, vp, vp, vp],
        "pk_weight_norm_bwd": [vp, vp, vp, i32, i32, vp, vp, vp],
        "pk_mse_const": [vp, i64, i32, i32, f32, vp, vp, f32, vp],
        "pk_sq_sum": [vp, i64, vp, vp],
        "pk_adam_clip": [vp, vp, vp, vp, i64, f32, f32, f32, f32, i32, vp, f32, vp],
        "pk_pwg_res_update": [vp, vp, i64, vp, i32, vp, vp, vp, vp],
        "pk_pwg_res_update_bwd": [vp, vp, i64, vp, vp, vp],
        "pk_up_stage_fwd": [vp, vp, i64, i32, i32, vp, vp],
        "pk_up_stage_bwd": [vp, vp, vp, i64, i32, i32, vp, vp, vp],
        "pk_stft_loss_grad": [vp, vp, vp, vp, i32, i32, i32, i32, vp, f32, vp, vp],
        "pk_frames_overlap_add": [vp, vp, i32, i32, i32, i32, i32, vp, vp],
        "pk_dropout": [vp, vp, vp, i64, f32, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp, vp, vp],
        "pk_waveflow_upsample": [vp, vp, vp, i32, i32, i32, i32, i32, f32, vp, vp],
        "pk_waveflow_input_proj": [vp, i64, vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, vp],
        "pk_gated_activation": [vp, i64, i32, vp, vp, vp],
        "pk_waveflow_layer_update": [vp, i64, i32, vp, vp, i32, vp, vp, i32, i32, vp],
        "pk_waveflow_row_out": [vp, vp, vp, vp, i64, i32, i32, i32, vp, i64, vp],
        "pk_spectral_loss_sums": [vp, vp, i64, f32, vp, vp],
        "pk_stft": [vp, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, i32, f32, vp, i32, vp, i32, f32, vp, f32, vp],
        "pk_waveflow_train_gather_split": [vp, vp, i64, vp, vp, vp],
        "pk_waveflow_train_input_fwd": [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp],
        "pk_waveflow_train_update": [vp, i32, i32, i32, i32, vp, vp, i32, vp, vp, vp],
        "pk_waveflow_train_tail_fwd": [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp],
        "pk_waveflow_forward_tail_bwd": [vp, vp, vp, vp, vp, vp, vp, f32, f32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, i32, vp],
        "pk_waveflow_train_input_bwd": [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp],
        "pk_waveflow_train_outer_sum": [vp, i32, i32, vp, i32, i32, i64, vp, i64, vp, i64, i64, i32, vp],
        "pk_waveflow_upsample_bwd": [vp, vp, vp, vp, i32, i32, i32, i32, f32, vp, vp, vp, i64, vp, vp, vp],
        "pk_waveflow_train_cond_gather": [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp],
        "pk_waveflow_train_cond_scatter": [vp, vp, i32, i32, i32, i32, i32, vp, vp],
        "pk_waveflow_train_loss": [vp, i64, vp, i64, f32, vp, vp],
        "pk_waveflow_backward_layer": [C.POINTER(WaveflowBackwardLayerArgs), vp],
        "pk_lstm_fwd": [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, i64, vp, vp, i64, vp],
        "pk_lstm_bwd": [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp],
        "pk_ge2e_loss": [vp, i32, i32, i32, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp],
        "pk_ge2e_embed_bwd": [vp, vp, i32, i32, f32, vp, vp],
        "pk_segment_mean_normalize": [vp, vp, i32, i32, f32, vp, vp],
        "pk_taco2_decode": [C.POINTER(Taco2DecodeArgs), vp],
        "pk_taco2_embed": [vp, vp, vp, vp, i32, i32, i32, vp, vp],
        "pk_taco2_time_major": [vp, vp, i32, i32, i32, i32, vp, vp],
        "pk_taco2_bilstm_merge": [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp],
        "pk_taco2_loss": [vp, vp, vp, i32, i32, i32, vp, i32, vp, vp, f32, vp, vp, vp],
        "pk_tts_decode": [C.POINTER(TtsDecodeArgs), vp],
        "pk_fused_attention_ex": [C.POINTER(AttentionArgs), vp],
        "pk_tts_text_eos": [vp, vp, i32, i32, i64, vp, vp],
        "pk_tts_shift_frames": [vp, i32, i32, i32, i32, vp, vp],
        "pk_tts_prenet_dropout": [vp, i32, i32, i32, f32, C.c_uint64, i32, vp],
        "pk_tts_stop_labels": [vp, i32, i32, vp, vp],
    }
    for name, argtypes in sigs.items():
        fn = getattr(L, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    L.pk_ge2e_loss_scratch.argtypes = [i32, i32, i32]
    L.pk_ge2e_loss_scratch.restype = i64
    L.pk_taco2_workspace.argtypes = [i32, i32, i32]
    L.pk_taco2_workspace.restype = i64
    L.pk_taco2_prof_len.argtypes = []
    L.pk_taco2_prof_len.restype = i64
    L.pk_tts_layer_floats.argtypes = [i32, i32]
    L.pk_tts_layer_floats.restype = i64
    L.pk_tts_workspace.argtypes = [i32, i32, i32, i32, i32]
    L.pk_tts_workspace.restype = i64


def check(rc, what=""):
    if rc != 0:
        msg = lib().pk_last_error().decode("utf-8", "replace")
        raise PkError(f"{what} failed with code {rc}: {msg}")


def launch_count():
    return int(lib().pk_launch_count())


def exported_symbols():
    """Names declared in include/parakeet_b200.h (used by the CPU-side symbol test)."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), "include", "parakeet_b200.h")
    text = open(hdr).read()
    return sorted(set(re.findall(r"^\s*(?:int|int64_t|const char\*)\s+(pk_\w+)\s*\(", text, flags=re.M)))
