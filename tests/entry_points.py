"""The ledger of the C entry points in include/omlm_b200.h: every symbol is either owned by the test file that checks
its correctness (OWNER) or listed as one the engine never launches, with the reason (NOT_LAUNCHED).

test_entry_points_cpu.py checks that the two maps cover the header exactly and that each owner file names its
symbols; test_entry_points_gpu.py runs every phase of tests/call_forms.py with lib.call patched and checks that what
the engine launches is owned, that nothing in NOT_LAUNCHED is launched, and that every owned symbol is launched."""

GEMM = "test_gemm_reference_gpu.py"
NORM_LOSS = "test_norm_loss_reference_gpu.py"
ATTN_FFN = "test_attention_ffn_call_forms_gpu.py"
SAMPLER_TOKEN = "test_sampler_token_call_forms_gpu.py"
RELPOS = "test_relpos_bias_gpu.py"
OPTIM = "test_optim_reference_gpu.py"
DATA = "test_data_gpu.py"
HOST = "host"           # host queries and workspace sizes: no kernel, nothing to check against a reference

OWNER = {
    # call-form inventories
    "omlm_gemm16": GEMM, "omlm_gemm16_splitk_det": GEMM, "omlm_gemm16_rowstat": GEMM, "omlm_skinny_gemm": GEMM,
    "omlm_decode_gemm": GEMM, "omlm_decode_gemm_invariant": GEMM,
    "omlm_layernorm_fwd": NORM_LOSS, "omlm_layernorm_bwd": NORM_LOSS, "omlm_layernorm_bwd_det": NORM_LOSS,
    "omlm_qk_l2norm_fwd": NORM_LOSS, "omlm_qk_l2norm_bwd": NORM_LOSS, "omlm_qk_l2norm_bwd_det": NORM_LOSS,
    "omlm_cross_entropy": NORM_LOSS, "omlm_cross_entropy_det": NORM_LOSS, "omlm_token_logprob": NORM_LOSS,
    "omlm_embed_gather": NORM_LOSS, "omlm_embed_scatter_add": NORM_LOSS, "omlm_embed_scatter_add_det": NORM_LOSS,
    "omlm_attn_fwd_tc": ATTN_FFN, "omlm_attn_bwd_tc": ATTN_FFN, "omlm_attn_bwd_tc_det": ATTN_FFN,
    "omlm_attn_fwd_tc_varlen": ATTN_FFN, "omlm_attn_fwd_tc_chunk": ATTN_FFN, "omlm_attn_decode_ragged": ATTN_FFN,
    "omlm_attn_decode_mqa_ragged": ATTN_FFN, "omlm_gemm_ffn_up": ATTN_FFN, "omlm_gemm_ffn_up_varlen": ATTN_FFN,
    "omlm_gemm_ffn_up_chunk": ATTN_FFN, "omlm_ffn_norm_fwd": ATTN_FFN, "omlm_ffn_mid_bwd": ATTN_FFN,
    "omlm_ffn_mid_bwd_det": ATTN_FFN, "omlm_decode_conv_geglu": ATTN_FFN,
    "omlm_sample_rows": SAMPLER_TOKEN, "omlm_sample_logprob": SAMPLER_TOKEN, "omlm_sample_rows_indexed": SAMPLER_TOKEN,
    "omlm_sample_rows_indexed_logprob": SAMPLER_TOKEN, "omlm_token_plan": SAMPLER_TOKEN, "omlm_forgetful_mask": SAMPLER_TOKEN,
    "omlm_embed_gather_pos_rows": SAMPLER_TOKEN, "omlm_decode_advance_pos": SAMPLER_TOKEN,
    # engine-level float64 tests
    "omlm_sgemm_small": RELPOS, "omlm_sgemm_small_det": RELPOS, "omlm_split3_bf16": RELPOS, "omlm_bias_silu": RELPOS,
    "omlm_silu_bwd": RELPOS, "omlm_colsum": RELPOS, "omlm_arange_f32": RELPOS,
    "omlm_grad_sumsq": OPTIM, "omlm_grad_sumsq_det": OPTIM, "omlm_adamw_step": OPTIM, "omlm_pack_multi": OPTIM,
    "omlm_gather_windows": DATA,
    "omlm_device_check": HOST, "omlm_num_sms": HOST, "omlm_last_error": HOST, "omlm_attn_bwd_tc_det_workspace": HOST,
    "omlm_decode_gemm_workspace": HOST, "omlm_decode_gemm_invariant_workspace": HOST,
}

# owned symbols that no phase of call_forms launches, and why that is right
OUTSIDE_PHASES = {
    "omlm_gather_windows": "the data loader's crop gather (data.TokenStore.sample_batch); the phases build their batches directly",
}

NOT_LAUNCHED = {
    "omlm_attn_fwd": "the attention forward of attn_fwd.cu; training, eval and prefill run attn_fwd_tc and its packed forms",
    "omlm_attn_bwd": "the attention backward of attn_bwd.cu; training runs attn_bwd_tc(_det)",
    "omlm_attn_decode": "the shared-position decode attention; every decode step passes per-row positions (_ragged)",
    "omlm_attn_decode_mqa": "the shared-position decode attention; every decode step passes per-row positions (_ragged)",
    "omlm_embed_gather_pos": "the shared-position gather; the decode step adds per-row positions (_pos_rows)",
    "omlm_embed_gather_pos_ragged": "the per-row-position gather without a per-row offset; the decode step uses _pos_rows",
    "omlm_sample": "the scalar sampler; generate and the stages pass per-row top-k and temperature (_rows, _logprob)",
    "omlm_sample_seeded": "the scalar seeded sampler; seeded generate passes per-row arguments (_rows, _logprob)",
    "omlm_sample_nucleus": "the scalar nucleus sampler; top_p reaches the kernel as per-row masses (_rows, _logprob)",
    "omlm_gemm_bf16": "the bf16-operand GEMM; lib has no wrapper for it and every GEMM goes through omlm_gemm16",
    "omlm_pack": "the one-job repack; the engine repacks every weight through PackTable (omlm_pack_multi)",
    "omlm_unpack_add": "the gradient unpack (lib.unpack_add); no module of the package calls it",
    "omlm_gemm16_splitk_det_workspace": "the split-K scratch size (lib.gemm_splitk_det_workspace); the engine sizes its "
                                        "deterministic partials itself",
    "omlm_abi_version": "the ABI number; lib has no wrapper for it, and test_boundary_cpu.py reads it from the library",
}

# the two host queries lib.py calls on the CDLL directly, not through lib.call
DIRECT_HOST_CALLS = {"omlm_last_error", "omlm_num_sms"}
