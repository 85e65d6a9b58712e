"""ctypes binding of ``libpcv_attn.so`` — the C-ABI declared in ``include/pcv_attn.h``.

The structures below mirror the header field by field (tests/test_abi.py checks the sizes and
that every declared symbol is exported).  There is deliberately no fallback: if the shared
library is missing the import of this module's :func:`lib` raises, and every op in
:mod:`perceiver_io_b200.ops` with it.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# PCV_LIB_PATH: developer override (A/B-testing two builds of the library on one GPU box)
LIB_PATH = os.environ.get("PCV_LIB_PATH") or os.path.join(_HERE, "lib", "libpcv_attn.so")

PCV_BF16, PCV_F16, PCV_F32, PCV_E4M3 = 0, 1, 2, 3
PCV_IMPL_AUTO, PCV_IMPL_TCGEN05, PCV_IMPL_SIMT, PCV_IMPL_TCGEN05_PAIR, PCV_IMPL_DECODE = 0, 1, 2, 3, 4
IMPL_BY_NAME = {"auto": PCV_IMPL_AUTO, "tcgen05": PCV_IMPL_TCGEN05, "simt": PCV_IMPL_SIMT, "decode": PCV_IMPL_DECODE,
                "tcgen05_pair": PCV_IMPL_TCGEN05_PAIR}

EXPORTS = (
    "pcv_abi_version",
    "pcv_last_error",
    "pcv_get_device_info",
    "pcv_attn_supported_tcgen05",
    "pcv_attn_workspace_bytes",
    "pcv_attn_fwd",
    "pcv_attn_combine",
    "pcv_attn_combine_peers",
    "pcv_attn_merge_partials",
    "pcv_attn_fwd_sharded_supported",
    "pcv_attn_fwd_sharded",
    "pcv_partial_rescale",
    "pcv_rotary_apply",
    "pcv_kv_append",
    "pcv_kv_project_supported",
    "pcv_ln_stats",
    "pcv_kv_project",
    "pcv_attn_bwd_supported",
    "pcv_attn_bwd_workspace_bytes",
    "pcv_attn_bwd",
    "pcv_attn_dropout_mask",
    "pcv_attn_dropout_mask_range",
    "pcv_attn_fwd_partial_dropout_supported",
    "pcv_attn_fwd_partial_dropout",
    "pcv_attn_fwd_partial_dropout_shard_supported",
    "pcv_attn_fwd_partial_dropout_shard",
    "pcv_attn_bwd_shard_supported",
    "pcv_attn_bwd_shard_workspace_bytes",
    "pcv_attn_bwd_shard",
    "pcv_attn_fwd_fp8_supported",
    "pcv_attn_fwd_fp8",
    "pcv_kv_project_fp8_supported",
    "pcv_kv_project_fp8",
    "pcv_attn_decode_fp8_supported",
    "pcv_attn_decode_fp8_workspace_bytes",
    "pcv_attn_decode_fp8",
    "pcv_attn_cached_fp8_supported",
    "pcv_attn_cached_fp8_workspace_bytes",
    "pcv_attn_cached_fp8",
    "pcv_kv_append_fp8_supported",
    "pcv_kv_append_fp8",
    "pcv_rotary_fp8_supported",
    "pcv_rotary_apply_fp8",
    "pcv_attn_decode_window_supported",
    "pcv_attn_decode_window_workspace_bytes",
    "pcv_attn_decode_window",
    "pcv_attn_decode_window_fp8_supported",
    "pcv_attn_decode_window_fp8",
    "pcv_attn_cached_window_supported",
    "pcv_attn_cached_window_workspace_bytes",
    "pcv_attn_cached_window",
    "pcv_attn_cached_window_fp8_supported",
    "pcv_attn_cached_window_fp8_workspace_bytes",
    "pcv_attn_cached_window_fp8",
    "pcv_kv_append_at",
    "pcv_kv_append_at_fp8",
    "pcv_rotary_apply_at",
    "pcv_rotary_apply_at_fp8",
    "pcv_sample_supported",
    "pcv_sample",
    "pcv_sample_uniforms",
    "pcv_spec_verify_supported",
    "pcv_spec_verify",
    "pcv_spec_uniforms",
    "pcv_beam_step_supported",
    "pcv_beam_step",
    "pcv_beam_step_logprobs_supported",
    "pcv_beam_step_logprobs",
    "pcv_logits_process_supported",
    "pcv_logits_process",
    "pcv_prompt_lookup_supported",
    "pcv_prompt_lookup",
    "pcv_kv_gather_rows_supported",
    "pcv_kv_gather_rows",
    "pcv_contrastive_candidates_supported",
    "pcv_contrastive_candidates",
    "pcv_contrastive_rank_supported",
    "pcv_contrastive_rank",
    "pcv_ln_linear_bwd_supported",
    "pcv_ln_linear_bwd_workspace_bytes",
    "pcv_ln_linear_bwd",
    "pcv_launch_count",
    "pcv_debug_plan",
    "pcv_debug_pair_workers",
    "pcv_profile_begin",
    "pcv_profile_end",
    "pcv_debug_read",
    "pcv_debug_trace_read",
)


class AttnParams(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("q_stride_b", C.c_int64), ("q_stride_n", C.c_int64), ("q_stride_h", C.c_int64),
        ("k_stride_b", C.c_int64), ("k_stride_m", C.c_int64), ("k_stride_h", C.c_int64),
        ("v_stride_b", C.c_int64), ("v_stride_m", C.c_int64), ("v_stride_h", C.c_int64),
        ("o_stride_b", C.c_int64), ("o_stride_n", C.c_int64), ("o_stride_h", C.c_int64),
        ("B", C.c_int32), ("H", C.c_int32), ("N", C.c_int32), ("M", C.c_int32),
        ("dqk", C.c_int32), ("dv", C.c_int32),
        ("scale", C.c_float),
        ("dtype", C.c_int32),
        ("causal", C.c_int32),
        ("m_total", C.c_int32),
        ("m_offset", C.c_int32),
        ("pad_mask", C.c_void_p),
        ("pad_stride_b", C.c_int64),
        ("write_partial", C.c_int32),
        ("part_o", C.c_void_p), ("part_m", C.c_void_p), ("part_l", C.c_void_p),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_size_t),
        ("impl", C.c_int32),
        ("reserved", C.c_int32),
    ]


class CombineParams(C.Structure):
    _fields_ = [
        ("part_o", C.c_void_p), ("part_m", C.c_void_p), ("part_l", C.c_void_p), ("out", C.c_void_p),
        ("o_stride_b", C.c_int64), ("o_stride_n", C.c_int64), ("o_stride_h", C.c_int64),
        ("num_parts", C.c_int32),
        ("B", C.c_int32), ("H", C.c_int32), ("N", C.c_int32), ("dv", C.c_int32),
        ("dtype", C.c_int32),
    ]


class MergeParams(C.Structure):
    _fields_ = [
        ("part_o", C.c_void_p), ("part_m", C.c_void_p), ("part_l", C.c_void_p),
        ("out_o", C.c_void_p), ("out_m", C.c_void_p), ("out_l", C.c_void_p),
        ("rows", C.c_int64), ("num_parts", C.c_int32), ("dv", C.c_int32),
    ]


PCV_MAX_PEERS = 8


class PeerCombineParams(C.Structure):
    _fields_ = [
        ("part_o", C.c_void_p * PCV_MAX_PEERS), ("part_m", C.c_void_p * PCV_MAX_PEERS),
        ("part_l", C.c_void_p * PCV_MAX_PEERS), ("out", C.c_void_p * PCV_MAX_PEERS),
        ("o_stride_b", C.c_int64), ("o_stride_n", C.c_int64), ("o_stride_h", C.c_int64),
        ("row_begin", C.c_int64), ("row_end", C.c_int64),
        ("num_peers", C.c_int32), ("rank", C.c_int32),
        ("B", C.c_int32), ("H", C.c_int32), ("N", C.c_int32), ("dv", C.c_int32),
        ("dtype", C.c_int32), ("reserved", C.c_int32),
    ]


class ShardFuse(C.Structure):
    _fields_ = [
        ("part", C.c_void_p * PCV_MAX_PEERS), ("out", C.c_void_p * PCV_MAX_PEERS), ("flags", C.c_void_p * PCV_MAX_PEERS),
        ("o_stride_b", C.c_int64), ("o_stride_n", C.c_int64), ("o_stride_h", C.c_int64),
        ("num_peers", C.c_int32), ("rank", C.c_int32), ("epoch", C.c_uint32), ("reserved", C.c_int32),
    ]


class RescaleParams(C.Structure):
    _fields_ = [
        ("part_o", C.c_void_p), ("part_m", C.c_void_p), ("part_l", C.c_void_p), ("new_m", C.c_void_p),
        ("rows", C.c_int64), ("dv", C.c_int32), ("reserved", C.c_int32),
    ]


class RotaryParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("y", C.c_void_p), ("angles", C.c_void_p),
        ("x_stride_b", C.c_int64), ("x_stride_n", C.c_int64), ("x_stride_h", C.c_int64),
        ("y_stride_b", C.c_int64), ("y_stride_n", C.c_int64), ("y_stride_h", C.c_int64),
        ("a_stride_b", C.c_int64), ("a_stride_n", C.c_int64),
        ("B", C.c_int32), ("n", C.c_int32), ("H", C.c_int32), ("d", C.c_int32),
        ("rotate_dim", C.c_int32),
        ("angle_row0", C.c_int32),
        ("dtype", C.c_int32),
        ("reserved", C.c_int32),
    ]


class KvAppendParams(C.Structure):
    _fields_ = [
        ("k_cache", C.c_void_p), ("v_cache", C.c_void_p),
        ("k_new", C.c_void_p), ("v_new", C.c_void_p),
        ("k_dst", C.c_void_p), ("v_dst", C.c_void_p),
        ("kc_stride_b", C.c_int64), ("kc_stride_l", C.c_int64), ("vc_stride_b", C.c_int64), ("vc_stride_l", C.c_int64),
        ("kn_stride_b", C.c_int64), ("kn_stride_l", C.c_int64), ("vn_stride_b", C.c_int64), ("vn_stride_l", C.c_int64),
        ("kd_stride_b", C.c_int64), ("kd_stride_l", C.c_int64), ("vd_stride_b", C.c_int64), ("vd_stride_l", C.c_int64),
        ("B", C.c_int32), ("L_old", C.c_int32), ("n", C.c_int32), ("Ck", C.c_int32), ("Cv", C.c_int32),
        ("dtype", C.c_int32),
    ]


class KvProjParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("col_st", C.c_void_p), ("row_stats", C.c_void_p),
        ("k_out", C.c_void_p), ("v_out", C.c_void_p),
        ("x_stride_row", C.c_int64), ("k_stride_row", C.c_int64), ("v_stride_row", C.c_int64),
        ("rows", C.c_int64),
        ("C", C.c_int32), ("n_k", C.c_int32), ("n_v", C.c_int32),
        ("dtype", C.c_int32), ("cta_group", C.c_int32), ("ln_eps", C.c_float),
    ]


class LnStatsParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("stats", C.c_void_p),
        ("x_stride_row", C.c_int64), ("rows", C.c_int64),
        ("C", C.c_int32), ("eps", C.c_float), ("dtype", C.c_int32), ("reserved", C.c_int32),
    ]


class AttnBwdParams(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p), ("grad_out", C.c_void_p),
        ("stat_m", C.c_void_p), ("stat_l", C.c_void_p),
        ("grad_q", C.c_void_p), ("grad_k", C.c_void_p), ("grad_v", C.c_void_p),
        ("q_stride_b", C.c_int64), ("q_stride_n", C.c_int64), ("q_stride_h", C.c_int64),
        ("k_stride_b", C.c_int64), ("k_stride_m", C.c_int64), ("k_stride_h", C.c_int64),
        ("v_stride_b", C.c_int64), ("v_stride_m", C.c_int64), ("v_stride_h", C.c_int64),
        ("o_stride_b", C.c_int64), ("o_stride_n", C.c_int64), ("o_stride_h", C.c_int64),
        ("go_stride_b", C.c_int64), ("go_stride_n", C.c_int64), ("go_stride_h", C.c_int64),
        ("gq_stride_b", C.c_int64), ("gq_stride_n", C.c_int64), ("gq_stride_h", C.c_int64),
        ("gk_stride_b", C.c_int64), ("gk_stride_m", C.c_int64), ("gk_stride_h", C.c_int64),
        ("gv_stride_b", C.c_int64), ("gv_stride_m", C.c_int64), ("gv_stride_h", C.c_int64),
        ("B", C.c_int32), ("H", C.c_int32), ("N", C.c_int32), ("M", C.c_int32),
        ("dqk", C.c_int32), ("dv", C.c_int32),
        ("scale", C.c_float), ("dtype", C.c_int32), ("causal", C.c_int32), ("dropout_p", C.c_float),
        ("dropout_seed", C.c_uint64),
        ("pad_mask", C.c_void_p), ("pad_stride_b", C.c_int64),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class KeyShard(C.Structure):
    _fields_ = [("m_total", C.c_int32), ("m_offset", C.c_int32), ("grad_q32", C.c_void_p)]


class Fp8Attn(C.Structure):
    _fields_ = [
        ("q_descale", C.c_void_p), ("k_descale", C.c_void_p), ("v_descale", C.c_void_p),
        ("vt_stride_b", C.c_int64), ("vt_stride_h", C.c_int64), ("vt_stride_c", C.c_int64),
        ("out_dtype", C.c_int32), ("reserved", C.c_int32),
    ]


class KvProjFp8(C.Structure):
    _fields_ = [
        ("inv_scale", C.c_void_p), ("vt_out", C.c_void_p),
        ("vt_stride_b", C.c_int64), ("vt_stride_h", C.c_int64), ("vt_stride_c", C.c_int64),
        ("keys_per_batch", C.c_int32), ("v_head_dim", C.c_int32),
    ]


class DecodeFp8(C.Structure):
    _fields_ = [("k_descale", C.c_void_p), ("v_descale", C.c_void_p)]


class KvFp8Scales(C.Structure):
    _fields_ = [("k_inv_scale", C.c_void_p), ("v_inv_scale", C.c_void_p)]


class RotaryFp8(C.Structure):
    _fields_ = [("x_descale", C.c_void_p), ("y_inv_scale", C.c_void_p)]


class DevRows(C.Structure):
    _fields_ = [("bounds", C.c_void_p), ("capacity", C.c_int32), ("bounds_stride_b", C.c_int32)]


SAMPLE_MAX_VOCAB = 32768   # PCV_SAMPLE_MAX_VOCAB


class SampleParams(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p), ("stride_row", C.c_int64),
        ("R", C.c_int32), ("V", C.c_int32), ("dtype", C.c_int32), ("rows_per_batch", C.c_int32),
        ("seeds", C.c_void_p), ("positions", C.c_void_p),
        ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("reserved", C.c_int32),
        ("tokens", C.c_void_p), ("logprobs", C.c_void_p),
    ]


SPEC_MAX_DRAFTS = 63   # PCV_SPEC_MAX_DRAFTS


class SpecVerifyParams(C.Structure):
    _fields_ = [
        ("target", C.c_void_p), ("t_stride_b", C.c_int64), ("t_stride_row", C.c_int64),
        ("draft", C.c_void_p), ("d_stride_b", C.c_int64), ("d_stride_row", C.c_int64),
        ("tokens", C.c_void_p), ("seeds", C.c_void_p), ("positions", C.c_void_p),
        ("B", C.c_int32), ("G", C.c_int32), ("V", C.c_int32),
        ("dtype", C.c_int32), ("draft_dtype", C.c_int32), ("reserved", C.c_int32),
        ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
        ("draft_temperature", C.c_float), ("draft_top_k", C.c_int32), ("draft_top_p", C.c_float),
        ("out_tokens", C.c_void_p), ("accepted", C.c_void_p),
    ]


BEAM_MAX_BEAMS = 8   # PCV_BEAM_MAX_BEAMS
BEAM_MAX_EOS = 4     # PCV_BEAM_MAX_EOS


class BeamStepParams(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p), ("stride_row", C.c_int64), ("length_penalty", C.c_double),
        ("B", C.c_int32), ("K", C.c_int32), ("V", C.c_int32), ("dtype", C.c_int32),
        ("n_eos", C.c_int32), ("eos", C.c_int32 * BEAM_MAX_EOS),
        ("early_stopping", C.c_int32), ("hist_len", C.c_int32),
        ("running_scores", C.c_void_p), ("finished_scores", C.c_void_p), ("finished_flags", C.c_void_p),
        ("running_hist", C.c_void_p), ("finished_hist", C.c_void_p), ("hist_scratch", C.c_void_p),
        ("item_flags", C.c_void_p), ("counters", C.c_void_p),
        ("cand_scores", C.c_void_p), ("cand_index", C.c_void_p),
        ("next_tokens", C.c_void_p), ("parents", C.c_void_p),
    ]


PROCESS_MAX_NGRAM = 8   # PCV_PROCESS_MAX_NGRAM
PROCESS_MAX_EOS = 4     # PCV_PROCESS_MAX_EOS


class LogitsProcessParams(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p), ("stride_row", C.c_int64), ("out", C.c_void_p), ("out_stride_row", C.c_int64),
        ("row_map", C.c_void_p), ("prefix", C.c_void_p), ("prefix_stride", C.c_int64),
        ("tail", C.c_void_p), ("tail_stride", C.c_int64), ("prefix_len", C.c_void_p), ("tail_len", C.c_void_p),
        ("prefix_len_stride", C.c_int32), ("tail_len_stride", C.c_int32),
        ("prefix_count", C.c_int32), ("prefix_cap", C.c_int32), ("tail_cap", C.c_int32),
        ("R", C.c_int32), ("V", C.c_int32), ("dtype", C.c_int32), ("row_group", C.c_int32), ("rows_per_hist", C.c_int32),
        ("log_softmax", C.c_int32), ("repetition_penalty", C.c_float), ("no_repeat_ngram", C.c_int32),
        ("min_new_tokens", C.c_int32), ("prompt_len", C.c_int32), ("n_eos", C.c_int32),
        ("eos", C.c_int32 * PROCESS_MAX_EOS),
    ]


LOOKUP_MAX_DRAFTS = 63   # PCV_LOOKUP_MAX_DRAFTS
LOOKUP_MAX_NGRAM = 16    # PCV_LOOKUP_MAX_NGRAM
LOOKUP_MAX_EOS = 4       # PCV_LOOKUP_MAX_EOS


class PromptLookupParams(C.Structure):
    _fields_ = [
        ("ids", C.c_void_p), ("ids_stride", C.c_int64), ("start", C.c_void_p), ("length", C.c_void_p),
        ("length_stride", C.c_int32), ("length_offset", C.c_int32), ("limit", C.c_void_p),
        ("B", C.c_int32), ("cap", C.c_int32), ("G", C.c_int32), ("N", C.c_int32), ("n_eos", C.c_int32),
        ("k", C.c_int32), ("eos", C.c_int64 * LOOKUP_MAX_EOS),
        ("drafts", C.c_void_p), ("drafts_stride", C.c_int64), ("counts", C.c_void_p), ("reserved", C.c_int32),
        ("fed", C.c_void_p), ("draws", C.c_void_p), ("t0", C.c_void_p), ("t0_stride", C.c_int64),
        ("accepted", C.c_void_p), ("unfinished", C.c_void_p), ("left", C.c_void_p),
    ]


class KvGatherEntry(C.Structure):
    _fields_ = [
        ("arena", C.c_void_p), ("scratch", C.c_void_p),
        ("arena_stride_b", C.c_int64), ("scratch_stride_b", C.c_int64),
        ("row_bytes", C.c_int32), ("first_row", C.c_int32), ("bounds_col", C.c_int32), ("max_rows", C.c_int32),
    ]


class KvGatherParams(C.Structure):
    _fields_ = [("table", C.c_void_p), ("n_entries", C.c_int32), ("R", C.c_int32), ("parents", C.c_void_p),
                ("last_rows", C.c_int32), ("reserved", C.c_int32)]


CONTRASTIVE_MAX_K = 16          # PCV_CONTRASTIVE_MAX_K
CONTRASTIVE_MAX_HIDDEN = 4096   # PCV_CONTRASTIVE_MAX_HIDDEN
CONTRASTIVE_MAX_EOS = 4         # PCV_CONTRASTIVE_MAX_EOS
CONTRASTIVE_ROWS_PER_CTA = 32   # PCV_CONTRASTIVE_ROWS_PER_CTA


class ContrastiveCandidatesParams(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p), ("stride_row", C.c_int64),
        ("B", C.c_int32), ("K", C.c_int32), ("V", C.c_int32), ("dtype", C.c_int32),
        ("sel", C.c_void_p), ("probs", C.c_void_p), ("cand", C.c_void_p), ("next_tokens", C.c_void_p),
    ]


class ContrastiveRankParams(C.Structure):
    _fields_ = [
        ("hidden", C.c_void_p), ("hidden_stride_row", C.c_int64), ("context", C.c_void_p),
        ("context_norm2", C.c_void_p), ("probs", C.c_void_p), ("cand", C.c_void_p),
        ("alpha", C.c_double), ("pad_token", C.c_int64),
        ("B", C.c_int32), ("K", C.c_int32), ("D", C.c_int32), ("hidden_dtype", C.c_int32),
        ("cap", C.c_int32), ("hist_len", C.c_int32), ("n_eos", C.c_int32), ("eos", C.c_int32 * CONTRASTIVE_MAX_EOS),
        ("reserved", C.c_int32),
        ("partial", C.c_void_p), ("sel", C.c_void_p), ("unfinished", C.c_void_p), ("history", C.c_void_p),
        ("counters", C.c_void_p), ("parents", C.c_void_p),
    ]


class LnLinearBwdParams(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("x_stride_row", C.c_int64), ("row_stats", C.c_void_p),
        ("w", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("grad_k", C.c_void_p), ("grad_v", C.c_void_p),
        ("gk_stride_row", C.c_int64), ("gv_stride_row", C.c_int64),
        ("grad_x", C.c_void_p), ("grad_w", C.c_void_p), ("grad_b", C.c_void_p),
        ("grad_gamma", C.c_void_p), ("grad_beta", C.c_void_p),
        ("rows", C.c_int64),
        ("C", C.c_int32), ("n_k", C.c_int32), ("n_v", C.c_int32), ("dtype", C.c_int32),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class DeviceInfo(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("sm_major", C.c_int32), ("sm_minor", C.c_int32),
        ("num_sms", C.c_int32), ("smem_optin_bytes", C.c_int32), ("tcgen05_ok", C.c_int32),
    ]


class PcvError(RuntimeError):
    """A libpcv_attn entry point returned a non-zero status."""


_lock = threading.Lock()
_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise PcvError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C perceiver_io_b200/csrc`). There is no CPU/PyTorch fallback for the attention path."
            )
        l = C.CDLL(LIB_PATH)
        l.pcv_abi_version.restype = C.c_int
        l.pcv_last_error.restype = C.c_char_p
        l.pcv_launch_count.restype = C.c_uint64
        l.pcv_get_device_info.argtypes = [C.POINTER(DeviceInfo)]
        l.pcv_attn_supported_tcgen05.argtypes = [C.POINTER(AttnParams)]
        l.pcv_attn_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_fwd.argtypes = [C.POINTER(AttnParams), C.c_void_p]
        l.pcv_attn_combine.argtypes = [C.POINTER(CombineParams), C.c_void_p]
        l.pcv_rotary_apply.argtypes = [C.POINTER(RotaryParams), C.c_void_p]
        l.pcv_partial_rescale.argtypes = [C.POINTER(RescaleParams), C.c_void_p]
        l.pcv_attn_combine_peers.argtypes = [C.POINTER(PeerCombineParams), C.c_void_p]
        l.pcv_attn_combine_peers.restype = C.c_int
        l.pcv_attn_merge_partials.argtypes = [C.POINTER(MergeParams), C.c_void_p]
        l.pcv_attn_merge_partials.restype = C.c_int
        l.pcv_attn_fwd_sharded_supported.argtypes = [C.POINTER(AttnParams)]
        l.pcv_attn_fwd_sharded_supported.restype = C.c_int
        l.pcv_attn_fwd_sharded.argtypes = [C.POINTER(AttnParams), C.POINTER(ShardFuse), C.c_void_p]
        l.pcv_attn_fwd_sharded.restype = C.c_int
        l.pcv_profile_begin.restype = C.c_int
        l.pcv_profile_end.restype = C.c_int
        l.pcv_profile_end.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_int32)]
        l.pcv_kv_append.argtypes = [C.POINTER(KvAppendParams), C.c_void_p]
        l.pcv_kv_project_supported.argtypes = [C.POINTER(KvProjParams)]
        l.pcv_kv_project_supported.restype = C.c_int
        l.pcv_ln_stats.argtypes = [C.POINTER(LnStatsParams), C.c_void_p]
        l.pcv_ln_stats.restype = C.c_int
        l.pcv_kv_project.argtypes = [C.POINTER(KvProjParams), C.c_void_p]
        l.pcv_kv_project.restype = C.c_int
        l.pcv_attn_bwd_supported.argtypes = [C.POINTER(AttnBwdParams)]
        l.pcv_attn_bwd_supported.restype = C.c_int
        l.pcv_attn_bwd_workspace_bytes.argtypes = [C.POINTER(AttnBwdParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_bwd_workspace_bytes.restype = C.c_int
        l.pcv_attn_bwd.argtypes = [C.POINTER(AttnBwdParams), C.c_void_p]
        l.pcv_attn_bwd.restype = C.c_int
        l.pcv_attn_dropout_mask.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                            C.c_uint64, C.c_void_p]
        l.pcv_attn_dropout_mask.restype = C.c_int
        l.pcv_attn_dropout_mask_range.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_float, C.c_uint64, C.c_void_p]
        l.pcv_attn_dropout_mask_range.restype = C.c_int
        l.pcv_attn_fwd_partial_dropout_supported.argtypes = [C.POINTER(AttnParams), C.c_float]
        l.pcv_attn_fwd_partial_dropout_supported.restype = C.c_int
        l.pcv_attn_fwd_partial_dropout.argtypes = [C.POINTER(AttnParams), C.c_float, C.c_uint64, C.c_void_p]
        l.pcv_attn_fwd_partial_dropout.restype = C.c_int
        l.pcv_attn_fwd_partial_dropout_shard_supported.argtypes = [C.POINTER(AttnParams), C.c_float]
        l.pcv_attn_fwd_partial_dropout_shard_supported.restype = C.c_int
        l.pcv_attn_fwd_partial_dropout_shard.argtypes = [C.POINTER(AttnParams), C.c_float, C.c_uint64, C.c_void_p]
        l.pcv_attn_fwd_partial_dropout_shard.restype = C.c_int
        l.pcv_attn_bwd_shard_supported.argtypes = [C.POINTER(AttnBwdParams), C.POINTER(KeyShard)]
        l.pcv_attn_bwd_shard_supported.restype = C.c_int
        l.pcv_attn_bwd_shard_workspace_bytes.argtypes = [C.POINTER(AttnBwdParams), C.POINTER(KeyShard),
                                                         C.POINTER(C.c_size_t)]
        l.pcv_attn_bwd_shard_workspace_bytes.restype = C.c_int
        l.pcv_attn_bwd_shard.argtypes = [C.POINTER(AttnBwdParams), C.POINTER(KeyShard), C.c_void_p]
        l.pcv_attn_bwd_shard.restype = C.c_int
        l.pcv_attn_fwd_fp8_supported.argtypes = [C.POINTER(AttnParams), C.POINTER(Fp8Attn)]
        l.pcv_attn_fwd_fp8_supported.restype = C.c_int
        l.pcv_attn_fwd_fp8.argtypes = [C.POINTER(AttnParams), C.POINTER(Fp8Attn), C.c_void_p]
        l.pcv_attn_fwd_fp8.restype = C.c_int
        l.pcv_kv_project_fp8_supported.argtypes = [C.POINTER(KvProjParams), C.POINTER(KvProjFp8)]
        l.pcv_kv_project_fp8_supported.restype = C.c_int
        l.pcv_kv_project_fp8.argtypes = [C.POINTER(KvProjParams), C.POINTER(KvProjFp8), C.c_void_p]
        l.pcv_kv_project_fp8.restype = C.c_int
        l.pcv_attn_decode_fp8_supported.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8)]
        l.pcv_attn_decode_fp8_supported.restype = C.c_int
        l.pcv_attn_decode_fp8_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_decode_fp8_workspace_bytes.restype = C.c_int
        l.pcv_attn_decode_fp8.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), C.c_void_p]
        l.pcv_attn_decode_fp8.restype = C.c_int
        l.pcv_attn_cached_fp8_supported.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8)]
        l.pcv_attn_cached_fp8_supported.restype = C.c_int
        l.pcv_attn_cached_fp8_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_cached_fp8_workspace_bytes.restype = C.c_int
        l.pcv_attn_cached_fp8.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), C.c_void_p]
        l.pcv_attn_cached_fp8.restype = C.c_int
        l.pcv_kv_append_fp8_supported.argtypes = [C.POINTER(KvAppendParams), C.POINTER(KvFp8Scales)]
        l.pcv_kv_append_fp8_supported.restype = C.c_int
        l.pcv_kv_append_fp8.argtypes = [C.POINTER(KvAppendParams), C.POINTER(KvFp8Scales), C.c_void_p]
        l.pcv_kv_append_fp8.restype = C.c_int
        l.pcv_rotary_fp8_supported.argtypes = [C.POINTER(RotaryParams), C.POINTER(RotaryFp8)]
        l.pcv_rotary_fp8_supported.restype = C.c_int
        l.pcv_rotary_apply_fp8.argtypes = [C.POINTER(RotaryParams), C.POINTER(RotaryFp8), C.c_void_p]
        l.pcv_rotary_apply_fp8.restype = C.c_int
        rows = C.POINTER(DevRows)
        l.pcv_attn_decode_window_supported.argtypes = [C.POINTER(AttnParams), rows]
        l.pcv_attn_decode_window_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_decode_window.argtypes = [C.POINTER(AttnParams), rows, C.c_void_p]
        l.pcv_attn_decode_window_fp8_supported.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), rows]
        l.pcv_attn_decode_window_fp8.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), rows, C.c_void_p]
        l.pcv_attn_cached_window_supported.argtypes = [C.POINTER(AttnParams), rows, C.c_int32]
        l.pcv_attn_cached_window_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_cached_window.argtypes = [C.POINTER(AttnParams), rows, C.c_int32, C.c_void_p]
        l.pcv_attn_cached_window_fp8_supported.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), rows, C.c_int32]
        l.pcv_attn_cached_window_fp8_workspace_bytes.argtypes = [C.POINTER(AttnParams), C.POINTER(C.c_size_t)]
        l.pcv_attn_cached_window_fp8.argtypes = [C.POINTER(AttnParams), C.POINTER(DecodeFp8), rows, C.c_int32,
                                                 C.c_void_p]
        l.pcv_kv_append_at.argtypes = [C.POINTER(KvAppendParams), rows, C.c_void_p]
        l.pcv_kv_append_at_fp8.argtypes = [C.POINTER(KvAppendParams), C.POINTER(KvFp8Scales), rows, C.c_void_p]
        l.pcv_rotary_apply_at.argtypes = [C.POINTER(RotaryParams), rows, C.c_void_p]
        l.pcv_rotary_apply_at_fp8.argtypes = [C.POINTER(RotaryParams), C.POINTER(RotaryFp8), rows, C.c_void_p]
        for name in ("pcv_attn_decode_window_supported", "pcv_attn_decode_window_workspace_bytes",
                     "pcv_attn_decode_window", "pcv_attn_decode_window_fp8_supported", "pcv_attn_decode_window_fp8",
                     "pcv_kv_append_at", "pcv_kv_append_at_fp8", "pcv_rotary_apply_at", "pcv_rotary_apply_at_fp8",
                     "pcv_attn_cached_window_supported", "pcv_attn_cached_window_workspace_bytes",
                     "pcv_attn_cached_window", "pcv_attn_cached_window_fp8_supported",
                     "pcv_attn_cached_window_fp8_workspace_bytes", "pcv_attn_cached_window_fp8"):
            getattr(l, name).restype = C.c_int
        l.pcv_sample_supported.argtypes = [C.POINTER(SampleParams)]
        l.pcv_sample.argtypes = [C.POINTER(SampleParams), C.c_void_p]
        l.pcv_sample_uniforms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        l.pcv_spec_verify_supported.argtypes = [C.POINTER(SpecVerifyParams)]
        l.pcv_spec_verify.argtypes = [C.POINTER(SpecVerifyParams), C.c_void_p]
        l.pcv_spec_uniforms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        for name in ("pcv_sample_supported", "pcv_sample", "pcv_sample_uniforms", "pcv_spec_verify_supported",
                     "pcv_spec_verify", "pcv_spec_uniforms"):
            getattr(l, name).restype = C.c_int
        l.pcv_beam_step_supported.argtypes = [C.POINTER(BeamStepParams)]
        l.pcv_beam_step.argtypes = [C.POINTER(BeamStepParams), C.c_void_p]
        l.pcv_kv_gather_rows_supported.argtypes = [C.POINTER(KvGatherParams), rows]
        l.pcv_kv_gather_rows.argtypes = [C.POINTER(KvGatherParams), rows, C.c_void_p]
        l.pcv_beam_step_logprobs_supported.argtypes = [C.POINTER(BeamStepParams)]
        l.pcv_beam_step_logprobs.argtypes = [C.POINTER(BeamStepParams), C.c_void_p]
        l.pcv_logits_process_supported.argtypes = [C.POINTER(LogitsProcessParams)]
        l.pcv_logits_process.argtypes = [C.POINTER(LogitsProcessParams), C.c_void_p]
        for name in ("pcv_beam_step_supported", "pcv_beam_step", "pcv_kv_gather_rows_supported", "pcv_kv_gather_rows",
                     "pcv_beam_step_logprobs_supported", "pcv_beam_step_logprobs", "pcv_logits_process_supported",
                     "pcv_logits_process"):
            getattr(l, name).restype = C.c_int
        l.pcv_prompt_lookup_supported.argtypes = [C.POINTER(PromptLookupParams)]
        l.pcv_prompt_lookup_supported.restype = C.c_int
        l.pcv_prompt_lookup.argtypes = [C.POINTER(PromptLookupParams), C.c_void_p]
        l.pcv_prompt_lookup.restype = C.c_int
        l.pcv_contrastive_candidates_supported.argtypes = [C.POINTER(ContrastiveCandidatesParams)]
        l.pcv_contrastive_candidates.argtypes = [C.POINTER(ContrastiveCandidatesParams), C.c_void_p]
        l.pcv_contrastive_rank_supported.argtypes = [C.POINTER(ContrastiveRankParams)]
        l.pcv_contrastive_rank.argtypes = [C.POINTER(ContrastiveRankParams), C.c_void_p]
        for name in ("pcv_contrastive_candidates_supported", "pcv_contrastive_candidates",
                     "pcv_contrastive_rank_supported", "pcv_contrastive_rank"):
            getattr(l, name).restype = C.c_int
        l.pcv_ln_linear_bwd_supported.argtypes = [C.POINTER(LnLinearBwdParams)]
        l.pcv_ln_linear_bwd_supported.restype = C.c_int
        l.pcv_ln_linear_bwd_workspace_bytes.argtypes = [C.POINTER(LnLinearBwdParams), C.POINTER(C.c_size_t)]
        l.pcv_ln_linear_bwd_workspace_bytes.restype = C.c_int
        l.pcv_ln_linear_bwd.argtypes = [C.POINTER(LnLinearBwdParams), C.c_void_p]
        l.pcv_ln_linear_bwd.restype = C.c_int
        l.pcv_debug_plan.argtypes = [C.c_int32] * 7 + [C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32)]
        l.pcv_debug_plan.restype = C.c_int
        l.pcv_debug_pair_workers.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        l.pcv_debug_pair_workers.restype = C.c_int
        for name in ("pcv_get_device_info", "pcv_attn_supported_tcgen05", "pcv_attn_workspace_bytes",
                     "pcv_attn_fwd", "pcv_attn_combine", "pcv_rotary_apply", "pcv_kv_append",
                     "pcv_partial_rescale"):
            getattr(l, name).restype = C.c_int
        if l.pcv_abi_version() != 2:
            raise PcvError(f"libpcv_attn ABI version {l.pcv_abi_version()} != 2 expected by the Python host")
        _lib = l
        return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().pcv_last_error()
        raise PcvError(f"{what} failed (status {rc}): {msg.decode() if msg else '?'}")


def profile_begin() -> None:
    check(lib().pcv_profile_begin(), "pcv_profile_begin")


def profile_end():
    """-> (summed device ms of the attention main kernel, number of launches) since profile_begin()."""
    ms, n = C.c_double(0.0), C.c_int32(0)
    check(lib().pcv_profile_end(C.byref(ms), C.byref(n)), "pcv_profile_end")
    return ms.value, n.value


def debug_read():
    """The tensor-core kernels' watchdog record (16 words; word 0 != 0 after a barrier-wait timeout)."""
    buf = (C.c_uint32 * 16)()
    l = lib()
    l.pcv_debug_read.restype = C.c_int
    l.pcv_debug_read.argtypes = [C.POINTER(C.c_uint32), C.c_int32]
    l.pcv_debug_read(buf, 16)
    return list(buf)


def debug_plan(B, H, N, M, workers=132, rows_per_unit=128):
    """Host-only: the tcgen05 work plan as (counts dict, list of (cta, b, h, q0, ntile, t0, t1, slot))."""
    counts = (C.c_int32 * 4)()
    lib().pcv_debug_plan(B, H, N, M, workers, rows_per_unit, 128, None, 0, counts)  # sizes only
    n = counts[0]
    segs = (C.c_int32 * (8 * max(n, 1)))()
    check(lib().pcv_debug_plan(B, H, N, M, workers, rows_per_unit, 128, segs, n, counts), "pcv_debug_plan")
    recs = [tuple(segs[8 * i + j] for j in range(8)) for i in range(n)]
    return {"segments": counts[0], "ctas": counts[1], "slots": counts[2], "units": counts[3]}, recs


def debug_pair_workers():
    """-> (CTA pairs of the current device's pair plan, 2-CTA clusters of the pair kernel that can be resident)."""
    w, fit = C.c_int32(0), C.c_int32(0)
    check(lib().pcv_debug_pair_workers(C.byref(w), C.byref(fit)), "pcv_debug_pair_workers")
    return w.value, fit.value


def launch_count() -> int:
    return int(lib().pcv_launch_count())
