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

#define OMLM_B200_ABI_VERSION 2
#define OMLM_MAX_SEQS 4

const char* omlm_last_error(void);
int omlm_abi_version(void);
/* 0 iff the current CUDA device is compute capability 10.x. */
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

/* ---- integer token path (bit-exact) ------------------------------------------------------------
 * One pass over the raw ids of all sequences of a TokenConditionedTransformer batch.
 * Wrapper mode (append_eos=1): eos (= codebook size) appended to every sequence
 * (open_musiclm.py:346-347, utils.py:112-117); labels = ids incl. eos (:355); drop_last drops the
 * predicted sequence's last token (:356); mask_cond masks + zeroes conditioning pad/eos ids
 * (:358-367).  Per position: row of the concatenated embedding table (offset = codebook_size *
 * (t mod q) added BEFORE the pad test, open_musiclm.py:126-133, utils.py:133-138; -1 = zero row;
 * start tokens are extra rows) and the key mask (AND mask_in AND forget_keep when given, :373-376).
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
int omlm_embed_scatter_add(float* dtable, const int* src_row, const float* dx, int M, int D,
                           float scale, void* stream);

/* ---- normalisation ------------------------------------------------------------------------------
 * Bias-less LayerNorm (transformer.py:24-31).  x fp32 [M,D] -> y [M,D] in fp16 (y_f16 = 1) or bf16 (row m written to row
 * dest_row[m] when given, skipped if negative), optional raw bf16 copy of x (keys/values are
 * projected from the un-normalised stream, transformer.py:228,254), stats[m] = (mean, rstd).  ycopy_bf16 (optional):
 * a bf16 copy of y for the weight-gradient GEMMs (one wgmma takes one operand format; gradients are bf16). */
int omlm_layernorm_fwd(const float* x, const float* gamma, void* y16, int y_f16, void* ycopy_bf16, void* xraw_bf16,
                       float* stats, const int* dest_row, int M, int D, void* stream);
/* dx = [dres] + [draw] + LN-backward(dy);  dgamma += sum_rows dy * xhat.  dy row for x row m is
 * src_row[m] when given (-1: no gradient).  dx_bf16 (optional): bf16 copy of dx for the next GEMMs. */
int omlm_layernorm_bwd(const void* dy_bf16, const float* x, const float* stats, const float* gamma,
                       const float* dres, const void* draw_bf16, const int* src_row, float* dx,
                       void* dx_bf16, float* dgamma, int M, int D, void* stream);
/* l2norm * learned scale on queries / keys (transformer.py:269-271, utils.py:68-69).
 * q_raw [M, heads*64], kv_raw [M,128] (k | v) -> qn, kvn (k normalised, v copied). */
int omlm_qk_l2norm_fwd(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale,
                       void* qn, void* kvn, int M, int heads, void* stream);
int omlm_qk_l2norm_bwd(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                       const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                       float* dq_scale, float* dk_scale, int M, int heads, void* stream);

/* ---- relative position bias MLP (transformer.py:36-67), fp32 SIMT ------------------------------
 * C[m,n] (+)= sum_k A[m*sa_m+k*sa_k] B[k*sb_k+n*sb_n] (+bias[n]); act 1 = SiLU (pre-activation to Z). */
int omlm_sgemm_small(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                     long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                     int accumulate, void* stream);
int omlm_silu_bwd(const float* dA, const float* Z, float* dZ, void* dZ_bf16, long n, void* stream);
/* bf16x3 operand split for near-fp32 products on the tensor cores: dst bf16 [R, 3C] = [hi|hi|lo] (activations)
 * or [hi|lo|hi] (weight_mode);  bias_silu: z += bias, a = silu(z). */
int omlm_split3_bf16(const float* src, long src_ld, void* dst, int R, int C, int weight_mode, void* stream);
int omlm_bias_silu(float* z, const float* bias, float* a, int R, int C, void* stream);
int omlm_colsum(const float* X, long s_m, long s_n, float* out, int M, int N, int accumulate, void* stream);
int omlm_arange_f32(float* out, int n, void* stream);

/* ---- attention (transformer.py:304-331, self-attention, causal, multi-query) -------------------
 * qn [B,N,heads*64] bf16, kvn [B,N,128] bf16, table fp32 [heads, table_ld] (bias for i-j >= 0),
 * key_mask u8 [B,N] or NULL -> out bf16 [B,N,heads*64], lse2 fp32 [B,N*heads] (log2 domain). */
int omlm_attn_fwd(const void* qn, const void* kvn, const float* table, int table_ld,
                  const unsigned char* key_mask, void* out, float* lse2, int B, int N, int heads,
                  float scale, void* stream);
/* Same contract on the wgmma/TMA path (one 128-row tile per CTA, two consumer warpgroups of 64 rows). */
int omlm_attn_fwd_tc(const void* qn, const void* kvn, const float* table, int table_ld,
                     const unsigned char* key_mask, void* out, float* lse2, int B, int N, int heads,
                     float scale, void* stream);
/* Accumulates (+=) into dqn fp32 [B,N,heads*64], dkvn fp32 [B,N,128], dtable fp32 [heads,table_ld]. */
int omlm_attn_bwd(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                  const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                  float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale,
                  void* stream);

/* wgmma/TMA backward: dqn and dkvn are OVERWRITTEN (its first kernel clears them, the main kernel reduces into
 * them), dtable is accumulated (+=: one table gradient over all layers).  The bias gradient -- diagonal sums of dS -- is
 * formed inside the kernel from the fp32 dS, summed per CTA in shared memory and added to dtable once; no scratch tensor.
 * dqn, dkvn and dtable are reduced with floating-point atomics: reproducible up to accumulation order. */
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
/* hn = dropout(LayerNorm_F(h)) from the fused statistics; stats fp32 [M, 2] = (mean, rstd) for the backward pass.
 * With drop_p > 0 the Philox keep mask is also written to keep_bits (uint8 [M, Fp/8], bit i of byte j = channel 8j+i)
 * so the backward pass reads 1 bit per element instead of regenerating the random stream. */
int omlm_ffn_norm_fwd(const void* h, const float* rowsum, const float* gamma, void* hn, void* hn_copy_bf16, float* stats,
                      void* keep_bits, long M, int F, int Fp, float drop_p, const unsigned long long* seed, int layer,
                      int act_f16, void* stream);
/* dhn, hn (saved forward output), keep_bits (from omlm_ffn_norm_fwd; may be NULL when drop_p == 0) -> du bf16 [B*N, 2Fp].
 * Parameter gradients are ACCUMULATED (+=) in the parameters' own layouts: dgamma [F] (inner LayerNorm gamma) and
 * dconv_w [2F, 3] (ds_conv.weight: value rows [0,F), gate rows [F,2F); may be NULL for the plain FeedForward).
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
 * vector, labels[r * label_stride]) -- the strided label view of one quantizer's logit-head group, read in place. */
int omlm_cross_entropy(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                       long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                       void* dlogits_bf16, long ldd, int Cp, float* loss_acc, void* stream);

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
/* CausalDSConv + GEGLU for one new row (transformer.py:122-137): u_new [B, 2Fp] against state [B, 2, 2Fp] (rows t-2, t-1,
 * shifted in place) -> h [B, Fp], rowsum [B, Fp/128, 2]. */
int omlm_decode_conv_geglu(const void* u_new, void* state, const float* conv_w, void* h_out, float* rowsum, int B, int Fp,
                           int act_f16, void* stream);
/* The whole incremental step in ONE launch (csrc/decode_fused.cu): embedding row, L x (q/kv projection, cached attention,
 * out-projection + residual, FFN-up + conv + GEGLU, inner LayerNorm + FFN-down + residual), final LayerNorm + the logit
 * head `w_logit` [C_pad, d] -> logits [B, ld_logits] fp32.  One CTA per SM with grid-wide barriers between the stages;
 * bit-identical to the sequence of omlm_embed_gather / omlm_skinny_gemm / omlm_attn_decode / omlm_decode_conv_geglu calls.
 * layers_device: DEVICE array of L records.  barrier: one device uint (zeroed by the call); err_flag is set to 1 if a
 * barrier times out (never hangs).  x0 (result), x1: fp32 [B, d] scratch; q_raw [B, heads*64], kv_raw [B, 128], o [B, heads*64]
 * bf16 scratch; hbuf [B, Fp] 16-bit and hf32 [B, Fp] fp32 scratch. */
typedef struct {
  const void *wq, *wkv, *wo, *w1, *w2;
  const float *conv, *gin, *g_attn, *g_ff, *q_scale, *k_scale;
  void* cache;
  void* conv_state;
} omlm_decode_layer;
int omlm_decode_step(const omlm_decode_layer* layers_device, int L, int B, int d, int heads, int F, int Fp, int n_max, int act_f16,
                     const float* emb_table, const int* next_row, const float* table, int table_ld, const int* pos_ptr,
                     float* x0, float* x1, void* q_raw, void* kv_raw, void* o, void* hbuf, float* hf32, const void* w_logit,
                     int C_pad, const float* g_final, float* logits, long ld_logits, unsigned int* barrier, int* err_flag,
                     float scale, void* stream);
/* Sampling of one token per sequence (open_musiclm.py:309-319, utils.py:71-84): eos (class C-1) forbidden unless
 * allow_eos, top-k with the given k, Gumbel-argmax at `temperature`.  uniform: optional [steps, B, C] uniform(0,1) draws
 * (slice *step_ptr is used; reproduces a given torch stream), else a Philox stream keyed by *seed.  Writes
 * tokens[b, *step_ptr] and next_row[b] = row_offset + token (embedding-table row for the next step), then advances
 * step_ptr[0] (step_ptr[1] is scratch) and, when given, pos_ptr[0]. */
int omlm_sample(const float* logits, long ld, int C, int top_k, float temperature, int allow_eos, const float* uniform,
                const unsigned long long* seed, long long* tokens, long tokens_ld, int* next_row, int row_offset, int* step_ptr,
                int* pos_ptr, int B, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OMLM_B200_H_ */
