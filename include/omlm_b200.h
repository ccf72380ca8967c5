/* libomlm_b200 — C ABI of the H100-native (sm_90a) hot path of zhvng/open-musiclm.
 *
 * The reference has no native code and therefore no FFI of its own: its hot path is the chain of
 * torch calls inside open_musiclm/transformer.py and open_musiclm/open_musiclm.py.  Each entry point
 * below replaces one such call site (cited as file:line relative to the reference tree).  All
 * functions
 *   - take only PODs (device pointers, sizes, float scalars, a cudaStream_t passed as void*),
 *   - are asynchronous (enqueue-only on the given stream) and allocate no persistent memory,
 *   - return 0 on success, 1 on argument errors, 1000+cudaError_t on CUDA errors;
 *     omlm_last_error() returns a thread-local description.
 * There is no CPU fallback: without an sm_90a device every compute entry point fails.
 */
#ifndef OMLM_B200_H_
#define OMLM_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define OMLM_B200_ABI_VERSION 4
#define OMLM_MAX_SEQS 4

const char* omlm_last_error(void);
int omlm_abi_version(void);
/* 0 iff the current CUDA device is compute capability 9.0. */
int omlm_device_check(void);
/* Number of SMs of the current device (the persistent kernels' default grid). */
int omlm_num_sms(void);

/* bf16 / fp16 GEMM on the wgmma tensor cores:  out[m,n] = alpha * sum_k A(m,k) * B(n,k) (+ addend[m,n]).
 *   a_mn_major = 0: A is [M, lda] with k contiguous;  1: A is [K, lda] with m contiguous.
 *   b_mn_major = 0: B is [N, ldb] with k contiguous;  1: B is [K, ldb] with n contiguous.
 *   out_f32: 0 -> bf16 out, 1 -> fp32 out.  addend (fp32, may alias out) gives residual add /
 *   beta=1 accumulation.  splits > 1: split-K with fp32 atomic accumulation into out.
 *   row_split/row_valid: output-row compaction for padded GEGLU weight layouts (0 = off; >0 two halves; <0 interleaved-128).
 *   n_valid: number of live output columns (<= N; 0 = N).  block_n in {128, 256}.
 * Replaces nn.Linear / einsum: transformer.py:144,149,254,333; open_musiclm.py:173,181 and their
 * autograd backward GEMMs. */
int omlm_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                   int M, int N, int K, void* out, int out_f32, long ldo, const float* addend,
                   long ldadd, float alpha, int splits, int row_split, int row_valid, int n_valid,
                   int block_n, int max_ctas, void* stream);
/* The same GEMM with the 16-bit operand format selectable: a_f16 = b_f16 = 1 -> IEEE fp16 operands, 0 -> bf16 (same
 * tensor rate, fp32 accumulation).  One wgmma instruction takes a single operand format, so
 * a_f16 != b_f16 is rejected.  The hot path uses fp16 for the forward GEMMs whose operands are bounded by
 * construction (LayerNorm outputs x weights, FFN activations) and bf16 wherever a gradient or the raw residual stream
 * is an operand. */
int omlm_gemm16(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major, long ldb,
                int M, int N, int K, void* out, int out_f32, long ldo, const float* addend,
                long ldadd, float alpha, int splits, int row_split, int row_valid, int n_valid,
                int block_n, int max_ctas, void* stream);

/* The same GEMM (dense bf16 output [M, N], 256-wide tiles, N % 256 == 0) whose epilogue also leaves, per output row and
 * 128-column half tile, the two row sums LayerNorm-backward needs against a saved tensor hn bf16 [M, N]:
 *   part[m, j, 0] = keep_scale * sum_{c in half tile j} gamma[c] * (keep_bit(m, c) ? d[m, c] : 0),
 *   part[m, j, 1] = sum_{c in half tile j} d[m, c] * hn[m, c],      j < parts = N / 128  (d = this GEMM's fp32 result).
 * Used for the d_hn data gradient of the conv feed-forward (transformer.py:140-150 backward): replaces a separate pass
 * over (dhn, hn).  keep_bits uint8 [M, N/8] or NULL. */
int omlm_gemm16_rowstat(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major, long ldb,
                        int M, int N, int K, void* out_bf16, long ldo, const void* hn_bf16, long ldhn, const void* keep_bits,
                        const float* gamma, float keep_scale, float* part, int parts, int max_ctas, void* stream);

/* ---- deterministic variants -------------------------------------------------------------------------------------
 * The training path's float reductions that the entry points above perform with atomics (so their results depend on
 * the order in which CTAs finish) have variants with the suffix _det.  Each keeps its default's contract and
 * arithmetic and fixes the order of every float sum, so repeated calls and CUDA-graph replays on one GPU model (same
 * SM count: tile and split choices depend on it) give bit-identical results.  Partial sums go to scratch the caller
 * owns (part_ws, part_ws_bytes: too small is an argument error); the library allocates nothing.
 *
 * Split-K GEMM, out fp32 += A B (the weight gradients): split s writes its fp32 partial [rows_out, ceil4(n_valid)] to
 * part_ws (no atomics) and a second kernel adds the partials to out in split order.  rows_out is the number of output
 * rows the row remap reaches (row_split > 0: M / row_split * row_valid, M must be a multiple of row_split; < 0:
 * 2 * row_valid; 0: M).  splits is
 * clamped as in omlm_gemm16; with one split the call is the in-place addend GEMM (no scratch used).
 * omlm_gemm16_splitk_det_workspace reports the bytes of part_ws (0 for one split). */
int omlm_gemm16_splitk_det(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major, long ldb,
                           int M, int N, int K, float* out, long ldo, int splits, int row_split, int row_valid, int n_valid,
                           int block_n, int max_ctas, float* part_ws, long part_ws_bytes, void* stream);
int omlm_gemm16_splitk_det_workspace(int M, int N, int K, int splits, int row_split, int row_valid, int n_valid, long* part_bytes);
/* omlm_layernorm_bwd: each CTA writes its dgamma sum as one row of part_ws (>= 4 * SMs * D floats), omlm_colsum adds
 * the rows to dgamma in CTA order.  dgamma == NULL: no partial rows, no omlm_colsum. */
int omlm_layernorm_bwd_det(const void* dy_bf16, const float* x, const float* stats, const float* gamma,
                           const float* dres, const void* draw_bf16, const int* src_row, float* dx,
                           void* dx_bf16, float* dgamma, int M, int D, float* part_ws, long part_ws_bytes, void* stream);
/* omlm_qk_l2norm_bwd: per-CTA rows of (q scale | k scale) sums in part_ws (>= 8 * SMs * 128 floats), then omlm_colsum
 * for each scale gradient that is not NULL (both NULL: no partial rows). */
int omlm_qk_l2norm_bwd_det(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                           const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                           float* dq_scale, float* dk_scale, int M, int heads, float* part_ws, long part_ws_bytes, void* stream);
/* omlm_ffn_mid_bwd: per-CTA rows [B * ceil(N / 128), 7F] of (dgamma [F] | dconv_w [2F, 3]) sums in part_ws, then
 * omlm_colsum; the part of a NULL output is neither written to part_ws nor summed. */
int omlm_ffn_mid_bwd_det(const void* dhn, const void* hn, const void* u, const float* stats, const float* conv_w,
                         const float* gamma, const void* keep_bits, float* rowstat, int rowstat_parts, void* du, float* dgamma,
                         float* dconv_w, int B, int N, int F, int Fp, float drop_p, int act_f16, float* part_ws, long part_ws_bytes,
                         void* stream);
/* omlm_sgemm_small without the split of K over CTAs (each output element is one CTA's in-order sum). */
int omlm_sgemm_small_det(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                         long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                         int accumulate, void* stream);
/* omlm_embed_scatter_add: each destination row is summed by one warp over its positions in ascending order
 * (dtable row + scale * dx rows, each add rounded).  first_ws: table_rows ints, INT_MAX before the first call (each call
 * leaves them so); rows outside [0, table_rows) are skipped. */
int omlm_embed_scatter_add_det(float* dtable, const int* src_row, const float* dx, int M, int D, float scale, int* first_ws,
                               int table_rows, void* stream);
/* omlm_cross_entropy: per-CTA (loss, rows) pairs in part_ws (>= ceil(rows / 8) * 8 bytes), added to loss_acc in CTA order
 * by omlm_colsum. */
int omlm_cross_entropy_det(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                           long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                           void* dlogits_bf16, long ldd, int Cp, float* loss_acc, float* part_ws, long part_ws_bytes, void* stream);
/* omlm_grad_sumsq: per-CTA double sums in part_ws (>= 4 * SMs doubles), added to acc in CTA order. */
int omlm_grad_sumsq_det(const float* g, long n, float prescale, double* acc, double* part_ws, long part_ws_bytes, void* stream);
/* omlm_attn_bwd_tc with a fixed order for dQ, dK|dV and the bias gradient: dQ of a row tile and dK|dV of a key tile are
 * added in turns (key tile, warpgroup) and (row chunk) kept by counters in iws; each CTA's diagonal sums go to its own
 * partial table in ws and a second kernel adds the tables to dtable in CTA order.  ws (ws_bytes) and iws (iws_count
 * ints) are sized by omlm_attn_bwd_tc_det_workspace (iws_count may be larger).  iws[iws_count - 1] is an error word that
 * must be zero before the first call.  It is set to 1 if a turn was not granted within seconds: the kernel never hangs,
 * and that call's sums -- and those of every later call until the caller clears the word -- are added in arrival order,
 * correct up to rounding like omlm_attn_bwd_tc's but not reproducible.  dtable == NULL: as omlm_attn_bwd_tc; ws is not
 * read (it may be NULL, ws_bytes 0), iws is still needed, and dqn / dkvn are bit-identical to the call with a table. */
int omlm_attn_bwd_tc_det(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                         const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                         float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale,
                         float* ws, long ws_bytes, int* iws, long iws_count, void* stream);
int omlm_attn_bwd_tc_det_workspace(int B, int N, int heads, long* ws_bytes, long* iws_count);

/* ---- integer token path (bit-exact) ------------------------------------------------------------
 * One pass over the raw ids of all sequences of a TokenConditionedTransformer batch.
 * Wrapper mode (append_eos=1): eos (= codebook size) appended to every sequence
 * (open_musiclm.py:346-347, utils.py:112-117); labels = ids incl. eos (:355); drop_last drops the
 * predicted sequence's last token (:356); mask_cond masks + zeroes conditioning pad/eos ids
 * (:358-367).  Per position: row of the concatenated embedding table (offset = codebook_size *
 * (t mod q) added BEFORE the pad test, open_musiclm.py:126-133, utils.py:133-138; -1 = zero row;
 * start tokens are extra rows) and the key mask: the conditioning pad/eos mask of mask_cond (1 elsewhere), or mask_in
 * instead when given (a self_attn_mask passed to the transformer itself, [B, N]), AND forget_keep when given (:373-376).
 *   ids[s]: int64 [B, len[s]] device pointers (host array of n_seqs pointers)
 *   ids_out int64 [B, sum n_tok]; src_row int32 [B, N]; key_mask u8 [B, N]; labels int32 [B, sum(len+eos)] or NULL.
 *   err_flag (device int, optional): bit s is set when sequence s holds an id outside its embedding table (where
 *   nn.Embedding would raise); such positions get the zero embedding instead of an out-of-bounds read. */
int omlm_token_plan(int n_seqs, const long long* const* ids, const int* len, const int* codebook,
                    const int* nq, const int* emb_row_base, const int* start_row, int B,
                    int append_eos, int drop_last, int mask_cond, int pad_id,
                    const unsigned char* mask_in, const unsigned char* forget_keep,
                    long long* ids_out, int* src_row, unsigned char* key_mask, int* labels,
                    int* err_flag, void* stream);
/* Forgetful causal mask (utils.py:49-56): keep[b,p]=0 for a uniformly random subset of num_drop
 * positions per row, never position 0.  seed: device pointer; stream_id separates draws. */
int omlm_forgetful_mask(unsigned char* keep, int B, int N, int num_drop,
                        const unsigned long long* seed, unsigned long long stream_id, void* stream);
/* x[m,:] = table[src_row[m],:] (+ table[src_row2[m],:] when src_row2 is given: the absolute position embeddings of
 * open_musiclm.py:134-136; negative rows add nothing) (fp32, 128-bit copies); replaces get_embeds + start-token concat
 * (open_musiclm.py:133-145).  scatter_add is its backward incl. the grad_shrink factor (utils.py:60-61). */
int omlm_embed_gather(const float* table, const int* src_row, const int* src_row2, float* x, int M, int D, void* stream);
/* The decode step's input rows with absolute position embeddings: x[m,:] = table[src_row[m],:] +
 * table[pos_row_base + p,:], p = *pos_ptr + pos_offset (pos_ptr: device int, read by the kernel so that a captured
 * CUDA graph uses the current position on every replay; one position row for all m).  A negative src_row, or p outside
 * [0, pos_rows), adds nothing (the caller checks the bound before launching).  fp32, 128-bit copies. */
int omlm_embed_gather_pos(const float* table, const int* src_row, const int* pos_ptr, int pos_offset, int pos_row_base,
                          int pos_rows, float* x, int M, int D, void* stream);
/* omlm_embed_gather_pos with one position per row, for prompts of different lengths in one batch: p = pos[m] +
 * pos_offset, pos a device int array [M].  The shared-position entry point above keeps its single read. */
int omlm_embed_gather_pos_ragged(const float* table, const int* src_row, const int* pos, int pos_offset, int pos_row_base,
                                 int pos_rows, float* x, int M, int D, void* stream);
/* omlm_embed_gather_pos_ragged with one predicted-sequence offset per row as well: p = pos[m] + pos_offset[m] (pos and
 * pos_offset device int arrays [M]), for the rows of a generation session, whose conditioning lengths differ. */
int omlm_embed_gather_pos_rows(const float* table, const int* src_row, const int* pos, const int* pos_offset, int pos_row_base,
                               int pos_rows, float* x, int M, int D, void* stream);
int omlm_embed_scatter_add(float* dtable, const int* src_row, const float* dx, int M, int D,
                           float scale, void* stream);

/* ---- normalisation ------------------------------------------------------------------------------
 * Bias-less LayerNorm (transformer.py:24-31).  x fp32 [M,D] -> y [M,D] in fp16 (y_f16 = 1) or bf16 (row m written to row
 * dest_row[m] when given, skipped if negative), optional raw bf16 copy of x (keys/values are
 * projected from the un-normalised stream, transformer.py:228,254), stats[m] = (mean, rstd).  ycopy_bf16 (optional):
 * a bf16 copy of y for the weight-gradient GEMMs (one wgmma takes one operand format; gradients are bf16). */
int omlm_layernorm_fwd(const float* x, const float* gamma, void* y16, int y_f16, void* ycopy_bf16, void* xraw_bf16,
                       float* stats, const int* dest_row, int M, int D, void* stream);
/* dx = [dres] + [draw] + LN-backward(dy);  dgamma += sum_rows dy * xhat (dgamma may be NULL: gamma frozen, not
 * summed).  dy row for x row m is src_row[m] when given (-1: no gradient).  dx_bf16 (optional): bf16 copy of dx for the
 * next GEMMs. */
int omlm_layernorm_bwd(const void* dy_bf16, const float* x, const float* stats, const float* gamma,
                       const float* dres, const void* draw_bf16, const int* src_row, float* dx,
                       void* dx_bf16, float* dgamma, int M, int D, void* stream);
/* l2norm * learned scale on queries / keys (transformer.py:269-271, utils.py:68-69).
 * q_raw [M, heads*64], kv_raw [M,128] (k | v) -> qn, kvn (k normalised, v copied). */
int omlm_qk_l2norm_fwd(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale,
                       void* qn, void* kvn, int M, int heads, void* stream);
/* dq_scale / dk_scale (+= sum dy * xhat over rows) may each be NULL: that scale is frozen and its sum is skipped. */
int omlm_qk_l2norm_bwd(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                       const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                       float* dq_scale, float* dk_scale, int M, int heads, void* stream);

/* ---- relative position bias MLP (transformer.py:36-67), fp32 SIMT ------------------------------
 * C[m,n] (+)= sum_k A[m*sa_m+k*sa_k] B[k*sb_k+n*sb_n] (+bias[n]); act 1 = SiLU (pre-activation to Z). */
int omlm_sgemm_small(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                     long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                     int accumulate, void* stream);
int omlm_silu_bwd(const float* dA, const float* Z, float* dZ, void* dZ_bf16, long n, void* stream);
/* bf16x3 operand split for near-fp32 products on the tensor cores: dst bf16 [R, 3 Cpad] = [hi|hi|lo] (activations)
 * or [hi|lo|hi] (weight_mode), each third Cpad >= C columns wide with zeros in [C, Cpad) (Cpad % 8 == 0 puts every
 * third on a 16-byte boundary);  bias_silu: z += bias, a = silu(z). */
int omlm_split3_bf16(const float* src, long src_ld, void* dst, int R, int C, int Cpad, int weight_mode, void* stream);
int omlm_bias_silu(float* z, const float* bias, float* a, int R, int C, void* stream);
int omlm_colsum(const float* X, long s_m, long s_n, float* out, int M, int N, int accumulate, void* stream);
int omlm_arange_f32(float* out, int n, void* stream);

/* ---- attention (transformer.py:304-331, self-attention, causal, multi-query) -------------------
 * qn [B,N,heads*64] bf16, kvn [B,N,128] bf16, table fp32 [heads, table_ld] (bias for i-j >= 0),
 * key_mask u8 [B,N] or NULL -> out bf16 [B,N,heads*64], lse2 fp32 [B,N*heads] (log2 domain). */
int omlm_attn_fwd(const void* qn, const void* kvn, const float* table, int table_ld,
                  const unsigned char* key_mask, void* out, float* lse2, int B, int N, int heads,
                  float scale, void* stream);
/* Same contract on the wgmma/TMA path (one 128-row tile per CTA, two consumer warpgroups of 64 rows; each reads the
 * bias from a per-tile window of the table staged in shared memory, so heads is limited to 68). */
int omlm_attn_fwd_tc(const void* qn, const void* kvn, const float* table, int table_ld,
                     const unsigned char* key_mask, void* out, float* lse2, int B, int N, int heads,
                     float scale, void* stream);
/* omlm_attn_fwd_tc over sequences of their own lengths packed back to back without padding (a packed prefill): qn
 * [M, heads*64], kvn [M, 128], out [M, heads*64], lse2 [M*heads] with M the packed rows.  Sequence b is rows
 * seq_start[b] .. seq_start[b] + seq_len[b] - 1 (int32 device arrays), causal within itself, without key mask; rows past
 * the last sequence are not written.  work (int32 device array [2 n_work]): one (sequence, 128-row query block of its
 * seq_len[b]*heads folded rows) pair per CTA, every block of every sequence once, heaviest first.  table_ld >= max_len
 * >= every seq_len[b].  Each CTA computes what omlm_attn_fwd_tc computes for that block with B = 1 and N = seq_len[b]:
 * out and lse2 are bit-identical to running each sequence alone. */
int omlm_attn_fwd_tc_varlen(const void* qn, const void* kvn, const float* table, int table_ld, const int* work, int n_work,
                            const int* seq_start, const int* seq_len, int M, int max_len, void* out, float* lse2, int heads,
                            float scale, void* stream);
/* omlm_attn_fwd_tc_varlen over chunks of longer sequences (a chunked prefill): sequence b's seq_len[b] query rows are
 * positions p0 = q_off[b] ... of its prompt (p0 * heads a multiple of 128) and its keys are rows kv_start[b] + j of kv
 * (kv_rows rows of 128, e.g. a K/V cache that already holds positions 0 .. p0 + seq_len[b] - 1), visible for
 * j < p0 + seq_len[b]; rows past that end may hold anything, NaN included.  work as above (row blocks counted from the
 * chunk's first row); table_ld >= max_end >= every p0 + seq_len[b].  out and lse2 of each chunk row are bit-identical to
 * omlm_attn_fwd_tc over the whole prompt. */
int omlm_attn_fwd_tc_chunk(const void* qn, const void* kv, long kv_rows, const float* table, int table_ld, const int* work,
                           int n_work, const int* seq_start, const int* seq_len, const int* q_off, const int* kv_start, int M,
                           int max_end, void* out, float* lse2, int heads, float scale, void* stream);
/* Accumulates (+=) into dqn fp32 [B,N,heads*64], dkvn fp32 [B,N,128], dtable fp32 [heads,table_ld]. */
int omlm_attn_bwd(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                  const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                  float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale,
                  void* stream);

/* wgmma/TMA backward: dqn and dkvn are OVERWRITTEN (its first kernel clears them, the main kernel reduces into
 * them), dtable is accumulated (+=: one table gradient over all layers).  The bias gradient -- diagonal sums of dS -- is
 * formed inside the kernel from the fp32 dS staged in shared memory (each thread sums its (head, diagonal) pairs in row
 * order, no shared-memory atomics), summed per CTA and added to dtable once; no scratch tensor.  The bias is read from a
 * per-tile window of the table in shared memory; the windows and diagonal tables limit heads to 58.
 * dqn, dkvn and dtable are reduced with floating-point atomics: reproducible up to accumulation order
 * (omlm_attn_bwd_tc_det fixes the order).  dtable == NULL (nothing trains the bias table): a kernel variant without the
 * fp32 dS staging and the diagonal sums runs; dqn and dkvn are computed in the same order as with a table. */
int omlm_attn_bwd_tc(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                     const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                     float* dqn, float* dkvn, float* dtable, int B, int N, int heads,
                     float scale, void* stream);

/* ---- ConvFeedForward (transformer.py:122-150) ---------------------------------------------------
 * Interleaved GEGLU layout: Fp = F rounded up to 128; u / W1 rows / conv taps are ordered in groups of 128 channels as
 * [128 value | 128 gate]; h / hn / gamma / W2 columns are in natural channel order (zero padded to Fp).
 * FFN up-projection GEMM (wgmma) with the causal depthwise conv (k=3), GEGLU (exact erf) and the LayerNorm row
 * statistics fused into its epilogue:  u bf16 [M, 2Fp], h bf16 [M, Fp], rowsum fp32 [M, Fp/128, 2] = per-128-channel
 * partial (sum h, sum h^2), plain stores (no zeroing needed; summed in a fixed order by omlm_ffn_norm_fwd).  M = B * Nseq rows, sequences of Nseq consecutive rows.
 * act_f16 = 1: xn, w1 are fp16 operands and the forward activations u, h, hn are fp16 (0: all bf16); the same flag
 * must be given to omlm_ffn_norm_fwd (h, hn) and omlm_ffn_mid_bwd (u).  Gradients (dhn, du) and the hn that
 * omlm_ffn_mid_bwd reads (omlm_ffn_norm_fwd's hn_copy_bf16 when act_f16) are always bf16. */
int omlm_gemm_ffn_up(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out, void* h_out,
                     float* rowsum, int M, int Nseq, int K, int Fp, int act_f16, int max_ctas, void* stream);
/* omlm_gemm_ffn_up over sequences of their own lengths packed back to back: row m's position within its sequence is
 * row_pos[m] (int32 device array [M]: 0, 1, 2, ... from each sequence's first row), which starts the conv history
 * afresh where M % Nseq did.  Every row's u, h and rowsum are bit-identical to omlm_gemm_ffn_up on its sequence alone. */
int omlm_gemm_ffn_up_varlen(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out, void* h_out,
                            float* rowsum, const int* row_pos, int M, int K, int Fp, int act_f16, int max_ctas, void* stream);
/* omlm_gemm_ffn_up_varlen over chunks that continue longer sequences: a row m with c = hist_idx[m] >= 0 (int32 device
 * array [M], -1 elsewhere) is the first row of a chunk at position p0 > 0, whose conv inputs t-2 and t-1 are rows 2c and
 * 2c + 1 of hist (pre-conv u rows of the sequence's positions p0 - 2 and p0 - 1, [*, 2 Fp] in the activation format; a
 * zero row for p0 - 2 < 0).  row_pos[m] is the row's position in its whole sequence.  Every row's u, h and rowsum are
 * bit-identical to omlm_gemm_ffn_up on the whole sequence. */
int omlm_gemm_ffn_up_chunk(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out, void* h_out,
                           float* rowsum, const int* row_pos, const void* hist, const int* hist_idx, int M, int K, int Fp,
                           int act_f16, int max_ctas, void* stream);
/* hn = dropout(LayerNorm_F(h)) from the fused statistics; stats fp32 [M, 2] = (mean, rstd) for the backward pass.
 * With drop_p > 0 the Philox keep mask is also written to keep_bits (uint8 [M, Fp/8], bit i of byte j = channel 8j+i)
 * so the backward pass reads 1 bit per element instead of regenerating the random stream. */
int omlm_ffn_norm_fwd(const void* h, const float* rowsum, const float* gamma, void* hn, void* hn_copy_bf16, float* stats,
                      void* keep_bits, long M, int F, int Fp, float drop_p, const unsigned long long* seed, int layer,
                      int act_f16, void* stream);
/* dhn, hn (saved forward output), keep_bits (from omlm_ffn_norm_fwd; may be NULL when drop_p == 0) -> du bf16 [B*N, 2Fp].
 * Parameter gradients are ACCUMULATED (+=) in the parameters' own layouts: dgamma [F] (inner LayerNorm gamma) and
 * dconv_w [2F, 3] (ds_conv.weight: value rows [0,F), gate rows [F,2F)).  Either may be NULL (frozen; dconv_w also for the
 * plain FeedForward): that sum is skipped.
 * rowstat: the LayerNorm-backward row sums (sum gamma*drop(dhn), sum dhn*hn) as fp32 [B*N, parts, 2]:
 *   rowstat_parts > 0: partial sums written by omlm_gemm16_rowstat (the d_hn GEMM's epilogue), parts = Fp / 128;
 *   rowstat_parts = 0: rowstat is a [B*N, 2] scratch and the sums are computed here by one extra pass over (dhn, hn). */
int omlm_ffn_mid_bwd(const void* dhn, const void* hn, const void* u, const float* stats, const float* conv_w,
                     const float* gamma, const void* keep_bits, float* rowstat, int rowstat_parts, void* du, float* dgamma,
                     float* dconv_w, int B, int N, int F, int Fp, float drop_p, int act_f16, void* stream);

/* ---- cross entropy (open_musiclm.py:401) --------------------------------------------------------
 * loss_acc[0] += loss_scale * sum of row losses, loss_acc[1] += rows counted; dlogits bf16 [rows, ldd] =
 * (softmax - onehot) * grad_scale, zero in columns [C, Cp).  The label of row r is
 * labels[(r / rows_per_batch) * batch_stride + (r % rows_per_batch) * label_stride] (rows_per_batch <= 0: one flat
 * vector, labels[r * label_stride]) -- the strided label view of one quantizer's logit-head group, read in place.
 * Any class count C >= 1.  C <= 1280 with Cp <= 1280 keeps each row in registers; above that the row is streamed twice
 * with 128-bit loads and 16-byte stores, which needs logits 16-byte aligned with ld % 4 == 0 and ld >= C, and (when
 * dlogits is given) dlogits 16-byte aligned with ldd % 8 == 0, Cp % 8 == 0 and C <= Cp <= ldd (argument errors
 * otherwise).  Both paths take 8 rows per CTA. */
int omlm_cross_entropy(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                       long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                       void* dlogits_bf16, long ldd, int Cp, float* loss_acc, void* stream);
/* Per-row log-probability of the label, out[r] = l[label_r] - logsumexp(row r) (fp32 [rows]): omlm_cross_entropy's row
 * loss, negated, from the same kernel bodies (labels, strided view and layout conditions as there; no gradient, no sum).
 * A label outside [0, C) gives 0.  Any C. */
int omlm_token_logprob(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch, long batch_stride,
                       int rows, int C, float* out, void* stream);

/* ---- optimiser (trainer.py:443-449, optimizer.py:3-34) ------------------------------------------
 * hyper (device, 9 floats): lr, beta1, beta2, eps, wd, 1-beta1^t, 1-beta2^t, max_grad_norm, grad prescale.
 * The arena is ordered [weight-decayed params | others]; n_decay = size of the first part. */
int omlm_grad_sumsq(const float* g, long n, float prescale, double* acc, void* stream);
int omlm_adamw_step(float* p, const float* g, float* m, float* v, long n, long n_decay, const float* hyper,
                    const double* sumsq, void* stream);
/* One launch for a whole table of omlm_pack jobs (the per-step refresh of the packed 16-bit weights).  The table is
 * DEVICE memory; unit_start = running sum of ceil(rows_p * ceil(cols_p/4) / 1024) over the preceding jobs,
 * total_units = that sum over all jobs.  njobs <= 512 per table.  dst_fmt: 0 = bf16, 1 = fp32, 2 = fp16.
 * dst2 (optional, NULL = none): a second destination of the same geometry in format dst2_fmt, written from the same
 * read of src (the forward GEMMs take fp16 copies of the matrices whose bf16 copies the backward GEMMs read). */
typedef struct {
  const float* src; void* dst; void* dst2;
  long src_ld, dst_ld, unit_start;
  int rows_valid, cols_valid, rows_p, cols_p, split_dst, split_src, dst_fmt, dst2_fmt;
} omlm_pack_job;
int omlm_pack_multi(const omlm_pack_job* jobs_device, int njobs, long total_units, void* stream);
/* canonical fp32 -> padded compute layout (bf16 or fp32) and gradient unpacking (+=). */
int omlm_pack(const float* src, long src_ld, int rows_valid, int cols_valid, void* dst, int dst_fmt, long dst_ld,
              int rows_p, int cols_p, int split_dst, int split_src, void* stream);
int omlm_unpack_add(const float* packed, long p_ld, int rows_p, int cols_p, float* dst, long dst_ld, int rows_valid,
                    int cols_valid, int split_dst, int split_src, void* stream);

/* ---- token store (open_musiclm/data.py:304-438: PreprocessedDataset crops) -----------------------------------------
 * out[b, t, c] = src[(start[b] + t) * width + c] (uint16 token ids widened to int64): one crop per batch row out of a
 * device-resident flat token array; `start` are rows (time steps), not elements. */
int omlm_gather_windows(const void* src_i16, const long long* start, long long* out, int len, int width, int B, void* stream);

/* ---- incremental (KV-cache) decoding: TokenConditionedTransformerWrapper.generate (open_musiclm.py:253-326) ----------
 * One new position per sequence and step instead of the reference's full-prefix forward per sampled token
 * (open_musiclm.py:303-307).  Batches of B <= 16 rows run the SIMT weight-streaming kernels of csrc/decode.cu
 * (omlm_skinny_gemm, omlm_attn_decode); 16 < B <= 256 run the tensor-core GEMM of csrc/decode_gemm.cu (omlm_decode_gemm)
 * and the cache-sharing attention omlm_attn_decode_mqa.
 * Every sequence is at the position the device int *pos_ptr holds; when the prompts of one batch differ in length, the
 * _ragged forms of the attention entry points (and omlm_embed_gather_pos_ragged) read one position per sequence from a
 * device int array pos [B] instead, and omlm_decode_advance_pos takes over the position bump from the sampler.
 * out[b, n] = A[b, :] . W[n, :] (+ addend[b, n]);  W 16-bit [N, ldw] (w_f16: fp16, else bf16).  prologue builds the
 * activation rows in W's format: 0 = A already 16-bit [B, lda];  1 = A fp32, rounded;  2 = LayerNorm(A fp32) * gamma
 * (transformer.py:24-31);  3 = A = h 16-bit [B, K] with the fused per-128-channel sums rowsum [B, K/128, 2]:
 * (h - mean) * rstd * gamma with n_real = F live channels (the inner LayerNorm of ConvFeedForward, transformer.py:147).
 * out_fmt: 0 bf16, 1 fp32, 2 fp16. */
int omlm_skinny_gemm(const void* A, long lda, int prologue, const void* W, long ldw, int w_f16, const float* gamma,
                     const float* rowsum, int n_real, const float* addend, long ldadd, void* out, int out_fmt, long ldo,
                     int B, int N, int K, void* stream);
/* The same contract for 1 <= B <= 256 rows on the wgmma tensor cores: the weight rows are the 64-row M operand, the batch
 * (padded to 64, 128 or 256) the N operand, and the K range is split over CTAs (fp32 partials, summed by a second
 * kernel in a fixed order) until the grid covers the SMs or the partials' bytes reach 4x the weights'.  Same
 * prologues with the same rounding points, same output formats and argument checks; the result differs from
 * omlm_skinny_gemm's only in the fp32 accumulation order.  Deterministic (no floating-point atomics): repeated calls and
 * CUDA-graph replays give bit-identical outputs.  out must not
 * overlap A.  Workspaces (device, owned by the caller, reusable by successive calls on one stream):
 *   a16_ws   16-byte aligned, B * K 16-bit elements: the activation operand (unused when prologue = 0 and A is 16-byte
 *            aligned with lda % 8 == 0: then A is read in place);
 *   part_ws  part_ws_bytes >= the part_bytes omlm_decode_gemm_workspace reports (split-K partials, fp32). */
int omlm_decode_gemm(const void* A, long lda, int prologue, const void* W, long ldw, int w_f16, const float* gamma,
                     const float* rowsum, int n_real, const float* addend, long ldadd, void* out, int out_fmt, long ldo,
                     int B, int N, int K, void* a16_ws, float* part_ws, long part_ws_bytes, void* stream);
/* Workspace omlm_decode_gemm needs for a B x N x K call (host-only query; depends on the current device's SM count). */
int omlm_decode_gemm_workspace(int B, int N, int K, long* part_bytes);
/* omlm_decode_gemm's contract with a K split that does not depend on B: the k-blocks per split are the ones
 * omlm_decode_gemm picks for a batch padded to 64 (a function of N, K and the SM count).  Row b of the output is then
 * bit-identical to the same row computed in a call of any other batch size, 1 to 256, on the same GPU model (seeded
 * generation relies on it).  Above 64 rows the split-K partials are up to 4x larger than omlm_decode_gemm's;
 * omlm_decode_gemm_invariant_workspace reports their bytes. */
int omlm_decode_gemm_invariant(const void* A, long lda, int prologue, const void* W, long ldw, int w_f16, const float* gamma,
                               const float* rowsum, int n_real, const float* addend, long ldadd, void* out, int out_fmt, long ldo,
                               int B, int N, int K, void* a16_ws, float* part_ws, long part_ws_bytes, void* stream);
int omlm_decode_gemm_invariant_workspace(int B, int N, int K, long* part_bytes);
/* Attention for the new position n = *pos_ptr (device int): q_raw [B, heads*64], kv_raw [B, 128] bf16 are this step's
 * un-normalised projections; they are l2-normalised * scale (transformer.py:269-271), [k | v] is appended to
 * cache [B, cache_ld_b/128 positions, 128] bf16 at n, then softmax(8 q.k_j + table[head, n-j]) V over keys 0..n
 * (transformer.py:304-331, no key mask: generate passes none).  max_pos bounds n + 1 (shared-memory scores). */
int omlm_attn_decode(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                     long cache_ld_b, const float* table, int table_ld, const int* pos_ptr, int max_pos, void* out, int B,
                     int heads, float scale, void* stream);
/* The same attention with every cached row read once per sequence (omlm_attn_decode reads it once per head): one CTA per
 * sequence and 128-key slice serves all heads (1 <= heads <= 16), and the slices are combined in a fixed order
 * (deterministic).  Same rounding points, except that P is rounded to bf16 relative to its slice's maximum: outputs
 * agree with omlm_attn_decode to bf16 rounding; the appended cache row is bit-identical.  Workspaces (device, owned by
 * the caller): ws fp32, ws_bytes >= B * ceil(max_pos / 128) * heads * 66 * 4;  counters B ints, ZERO before the first
 * call (each call leaves them zero). */
int omlm_attn_decode_mqa(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                         long cache_ld_b, const float* table, int table_ld, const int* pos_ptr, int max_pos, void* out, int B,
                         int heads, float scale, float* ws, long ws_bytes, int* counters, void* stream);
/* omlm_attn_decode and omlm_attn_decode_mqa with one position per sequence: sequence b appends its [k | v] at n = pos[b]
 * and attends over its keys 0..pos[b] with bias deltas pos[b] - j (pos: device int array [B], each entry < max_pos).  In
 * the _mqa form a sequence uses the slices its own n covers, counts its arrivals and combines them in slice order exactly
 * as it would alone, so its output is bit-identical to the same sequence in a call with B = 1. */
int omlm_attn_decode_ragged(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                            long cache_ld_b, const float* table, int table_ld, const int* pos, int max_pos, void* out, int B,
                            int heads, float scale, void* stream);
int omlm_attn_decode_mqa_ragged(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                                long cache_ld_b, const float* table, int table_ld, const int* pos, int max_pos, void* out, int B,
                                int heads, float scale, float* ws, long ws_bytes, int* counters, void* stream);
/* Per-sequence position bump of a decode step whose prompts differ in length (the sampler is then called with
 * pos_ptr = NULL): pos[b] += 1 while pos[b] < pos_last[b], the last position sequence b processes.  A sequence that
 * has all its tokens keeps its position, so one captured step serves every step of the call.  Device int arrays [B]. */
int omlm_decode_advance_pos(int* pos, const int* pos_last, int B, void* stream);
/* CausalDSConv + GEGLU for one new row (transformer.py:122-137): u_new [B, 2Fp] against state [B, 2, 2Fp] (rows t-2, t-1,
 * shifted in place) -> h [B, Fp], rowsum [B, Fp/128, 2]. */
int omlm_decode_conv_geglu(const void* u_new, void* state, const float* conv_w, void* h_out, float* rowsum, int B, int Fp,
                           int act_f16, void* stream);
/* Sampling of one token per sequence (open_musiclm.py:309-319, utils.py:71-84): eos (class C-1) forbidden unless
 * allow_eos, top-k with the given k (exactly k kept: among values equal to the k-th largest the lower indices win, and
 * -0.0 equals +0.0), Gumbel-argmax at `temperature`; 2 <= C <= 16384.  uniform: optional [steps, B, C] uniform(0,1) draws
 * (slice *step_ptr is used; reproduces a given torch stream), else a Philox stream keyed by *seed.  Writes
 * tokens[b, *step_ptr] and next_row[b] = row_offset + token (embedding-table row for the next step), then advances
 * step_ptr[0] (step_ptr[1] is scratch) and, when given, pos_ptr[0]. */
int omlm_sample(const float* logits, long ld, int C, int top_k, float temperature, int allow_eos, const float* uniform,
                const unsigned long long* seed, long long* tokens, long tokens_ld, int* next_row, int row_offset, int* step_ptr,
                int* pos_ptr, int B, void* stream);
/* omlm_sample with per-sequence seeds (device, B unsigned 64-bit values; NULL: omlm_sample).  The uniform of class c at
 * sample index t = *step_ptr of sequence b is word x0 of Philox-4x32-7 on the counter (c, t, 0, 0x5eed) under the key
 * seeds[b] (low word first), as (x0 >> 8) / 2^24: it does not depend on b or B.  seeds and uniform exclude each other;
 * seed is then unused. */
int omlm_sample_seeded(const float* logits, long ld, int C, int top_k, float temperature, int allow_eos, const float* uniform,
                       const unsigned long long* seed, const unsigned long long* seeds, long long* tokens, long tokens_ld,
                       int* next_row, int row_offset, int* step_ptr, int* pos_ptr, int B, void* stream);
/* Nucleus (top-p, Holtzman et al. 2019) sampling on top of omlm_sample / omlm_sample_seeded, 0 < top_p < 1 (anything
 * else is rejected).  For one row: eos and the top-k set K as in omlm_sample; p_c = softmax(l / temperature) over K, the
 * distribution the Gumbel-argmax samples from; the nucleus is
 *     N = { c in K : sum of p_j over j in K with l_j > l_c  <  top_p }
 * -- the smallest prefix of K by value whose mass reaches top_p, with equal values all in N or all out; the most likely
 * value is always in N.  The token is the argmax over N of l_c / temperature + g_c, with g_c drawn from the same uniform
 * the other samplers would use for class c (supplied, Philox keyed by *seed, or by seeds[b] when seeds is not NULL;
 * seeds and uniform exclude each other).  A NaN logit is never in N and has no mass; a row whose maximum over K is not
 * finite samples as omlm_sample does.  The sums behind N run in a fixed order, so a row's token does not depend on the
 * batch or the row.  Counters and outputs as omlm_sample. */
int omlm_sample_nucleus(const float* logits, long ld, int C, int top_k, float temperature, float top_p, int allow_eos,
                        const float* uniform, const unsigned long long* seed, const unsigned long long* seeds, long long* tokens,
                        long tokens_ld, int* next_row, int row_offset, int* step_ptr, int* pos_ptr, int B, void* stream);
/* The samplers above with sampling arguments per sequence (a batch whose rows are independent requests, or one prompt
 * at several settings).  top_k_rows (int [B]), temperature_rows and top_p_rows (float [B]) are optional device arrays;
 * where one is given, sequence b uses element b, otherwise the scalar top_k / temperature (checked as in omlm_sample).
 * A row's k is clamped to [1, C]; a row whose top_p lies outside (0, 1), NaN included, is not narrowed to a nucleus.
 * With top_p_rows the nucleus kernel runs (3 C floats of shared memory instead of 2), without it the plain one; a row
 * that is not narrowed samples bit-identically to omlm_sample_seeded with its own k and temperature, and a row with
 * top_p in (0, 1) to omlm_sample_nucleus.  The values reach the arithmetic as the scalar entry points take them, so a
 * row's token equals the token a call with that row's scalars gives.  Any value in the arrays keeps every access in
 * bounds.  uniform, seed, seeds, counters and outputs as omlm_sample_seeded. */
int omlm_sample_rows(const float* logits, long ld, int C, int top_k, const int* top_k_rows, float temperature,
                     const float* temperature_rows, const float* top_p_rows, int allow_eos, const float* uniform,
                     const unsigned long long* seed, const unsigned long long* seeds, long long* tokens, long tokens_ld,
                     int* next_row, int row_offset, int* step_ptr, int* pos_ptr, int B, void* stream);
/* omlm_sample_rows with one sample index per sequence, for a generation session whose rows joined at different steps:
 * sequence b reads t = step_rows[b] (device int [B]) in place of the shared counter, draws from Philox on the counter
 * (c, t, 0, 0x5eed) under seeds[b] (required; no supplied uniforms), writes tokens[b, t] and next_row[b], and sets
 * step_rows[b] = t + 1.  A sequence with t outside [0, min(n_rows[b], tokens_ld)) (n_rows: device int [B], the number
 * of tokens sequence b samples) writes nothing and keeps t.  Positions are not advanced (omlm_decode_advance_pos).
 * Per-row arrays, kernel choice and arithmetic as omlm_sample_rows: with every t equal, its tokens are bit-identical
 * to omlm_sample_rows with seeds at that sample index. */
int omlm_sample_rows_indexed(const float* logits, long ld, int C, int top_k, const int* top_k_rows, float temperature,
                             const float* temperature_rows, const float* top_p_rows, int allow_eos, const unsigned long long* seeds,
                             long long* tokens, long tokens_ld, int* next_row, int row_offset, int* step_rows, const int* n_rows,
                             int B, void* stream);
/* Token log-probabilities beside the token (float [B, tokens_ld] device arrays, written at the token's [b, t]).  They
 * share the tokens' allocation: logprobs must start right after tokens' B rows (at tokens + B * tokens_ld, read as
 * float) and sample_logprobs right after logprobs (logprobs + B * tokens_ld); anything else is an argument error.  The
 * pointers are checked, not passed to the kernel, so the samplers without log-probabilities keep their code.
 *   logprobs[b, t]        = l_c - (m + log sum_j exp(l_j - m)), over the raw row (all C classes, eos included, before
 *                           eos masking, temperature, top-k and top-p; m = its maximum): the model's log p of the token;
 *   sample_logprobs[b, t] = (l_c - m_S) / T - log sum_{j in S} exp((l_j - m_S) / T): its log p under the distribution
 *                           it was drawn from, S the candidate set (eos rule, top-k set K, then the nucleus N when the
 *                           row is narrowed); NaN entries are never in S, -inf entries add no mass.
 * The sums run in a fixed order (double accumulators of expf terms), so both values depend only on the row.  Tokens,
 * counters and every other argument as omlm_sample_rows (top_k_rows, temperature_rows, top_p_rows may be NULL; the
 * nucleus kernel runs when top_p_rows is given or the scalar top_p, in (0, 1], is below 1): the tokens are bit-identical
 * to the entry points without log-probabilities. */
int omlm_sample_logprob(const float* logits, long ld, int C, int top_k, const int* top_k_rows, float temperature,
                        const float* temperature_rows, float top_p, const float* top_p_rows, int allow_eos, const float* uniform,
                        const unsigned long long* seed, const unsigned long long* seeds, long long* tokens, long tokens_ld,
                        int* next_row, int row_offset, int* step_ptr, int* pos_ptr, int B, float* logprobs,
                        float* sample_logprobs, void* stream);
/* omlm_sample_rows_indexed with the two log-probabilities of omlm_sample_logprob, written at [b, step_rows[b]] by the
 * rows that sample. */
int omlm_sample_rows_indexed_logprob(const float* logits, long ld, int C, int top_k, const int* top_k_rows, float temperature,
                                     const float* temperature_rows, const float* top_p_rows, int allow_eos,
                                     const unsigned long long* seeds, long long* tokens, long tokens_ld, int* next_row,
                                     int row_offset, int* step_rows, const int* n_rows, int B, float* logprobs,
                                     float* sample_logprobs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OMLM_B200_H_ */
