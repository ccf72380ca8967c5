// Integer token path + embedding gather/scatter (bit-exact contract).
//
// Replaces, in one pass over the ids:
//   TokenConditionedTransformerWrapper.forward pre-processing  open_musiclm/open_musiclm.py:336-376
//   append_eos_id / generate_mask_with_prob                    open_musiclm/utils.py:112-117, 49-56
//   offsets + get_embeds + start-token interleave               open_musiclm/open_musiclm.py:123-145, utils.py:126-143
#include "common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

struct TokenPlanArgs {
  const long long* ids[OMLM_MAX_SEQS];  // raw ids [B, len]
  int len[OMLM_MAX_SEQS];
  int codebook[OMLM_MAX_SEQS];
  int nq[OMLM_MAX_SEQS];
  int emb_row_base[OMLM_MAX_SEQS];  // first row of embeddings[s] in the concatenated table
  int start_row[OMLM_MAX_SEQS];     // row of start_tokens[s] in the concatenated table
  int n_seqs;
  int append_eos;     // wrapper mode: eos (= codebook size) appended to every sequence
  int drop_last;      // return_loss: the predicted sequence loses its last token (the eos)
  int mask_cond;      // wrapper mode: conditioning pad/eos ids masked out of attention and zeroed
  int pad_id;
};

// One block per batch row.
__global__ void token_plan_kernel(const TokenPlanArgs a, const unsigned char* __restrict__ mask_in,
                                  const unsigned char* __restrict__ forget_keep,
                                  long long* __restrict__ ids_out, int* __restrict__ src_row,
                                  unsigned char* __restrict__ key_mask, int* __restrict__ labels,
                                  int* __restrict__ err_flag, int N, int n_ids_total, int n_labels_total) {
  const int b = blockIdx.x;
  int pos = 0, id_off = 0, lab_off = 0;
  for (int s = 0; s < a.n_seqs; ++s) {
    const bool last = (s == a.n_seqs - 1);
    const int len = a.len[s];
    const int n_with_eos = len + (a.append_eos ? 1 : 0);
    const int n_tok = n_with_eos - ((last && a.drop_last) ? 1 : 0);
    const long long eos = a.codebook[s];
    const long long* src = a.ids[s] + static_cast<long long>(b) * len;
    // labels = ids after eos append, before the drop and before the in-place zeroing (:355)
    if (labels != nullptr) {
      for (int t = threadIdx.x; t < n_with_eos; t += blockDim.x)
        labels[static_cast<long long>(b) * n_labels_total + lab_off + t] =
            static_cast<int>(t < len ? src[t] : eos);
    }
    if (threadIdx.x == 0) {  // start token slot
      src_row[static_cast<long long>(b) * N + pos] = a.start_row[s];
      unsigned char m = 1;
      if (mask_in != nullptr) m = mask_in[static_cast<long long>(b) * N + pos];
      if (forget_keep != nullptr) m = m && forget_keep[static_cast<long long>(b) * N + pos];
      key_mask[static_cast<long long>(b) * N + pos] = m;
    }
    for (int t = threadIdx.x; t < n_tok; t += blockDim.x) {
      long long id = t < len ? src[t] : eos;
      unsigned char m = 1;
      if (a.mask_cond && !last) {
        m = (id != a.pad_id) && (id != eos);  // :361
        if (!m) id = 0;                       // :363
      }
      ids_out[static_cast<long long>(b) * n_ids_total + id_off + t] = id;
      long long c = id;
      if (a.nq[s] > 1) c += static_cast<long long>(a.codebook[s]) * (t % a.nq[s]);  // :126-130
      const bool pad = (c == a.pad_id);                                               // utils.py:133
      const int p = pos + 1 + t;
      // nn.Embedding raises on an index outside [0, (codebook+1) * q): here the row is dropped (zero embedding, no
      // out-of-bounds read) and the error is latched in err_flag for the host to raise at its next synchronisation
      const bool oob = !pad && (c < 0 || c >= (static_cast<long long>(a.codebook[s]) + 1) * a.nq[s]);
      if (oob && err_flag != nullptr) atomicOr(err_flag, 1 << s);
      src_row[static_cast<long long>(b) * N + p] = (pad || oob) ? -1 : a.emb_row_base[s] + static_cast<int>(c);
      if (mask_in != nullptr) m = mask_in[static_cast<long long>(b) * N + p];
      if (forget_keep != nullptr) m = m && forget_keep[static_cast<long long>(b) * N + p];
      key_mask[static_cast<long long>(b) * N + p] = m;
    }
    pos += 1 + n_tok;
    id_off += n_tok;
    lab_off += n_with_eos;
  }
}

// Forgetful causal mask (utils.py:49-56): per row drop a uniformly random subset of
// min(int(N*p), N-1) positions, never position 0.  keep[b, p] = 1 if kept.
// One block per row; rank of each position's Philox key by counting (N <= a few thousand).
__global__ void forgetful_mask_kernel(unsigned char* __restrict__ keep, int N, int num_drop,
                                      const unsigned long long* __restrict__ seed_ptr,
                                      unsigned long long stream_id) {
  extern __shared__ unsigned int keys[];
  const int b = blockIdx.x;
  const unsigned long long seed = *seed_ptr;
  for (int p = threadIdx.x; p < N; p += blockDim.x) {
    const uint4 r = philox4x32(static_cast<uint32_t>(p), static_cast<uint32_t>(b),
                               static_cast<uint32_t>(stream_id), static_cast<uint32_t>(stream_id >> 32),
                               static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
    keys[p] = (p == 0) ? 0u : (r.x | 1u);  // position 0 gets the minimum key: never among the top
  }
  __syncthreads();
  for (int p = threadIdx.x; p < N; p += blockDim.x) {
    const unsigned int k = keys[p];
    int rank = 0;  // number of positions with a strictly larger key (ties broken by index)
    for (int j = 0; j < N; ++j) {
      const unsigned int kj = keys[j];
      rank += (kj > k) || (kj == k && j < p);
    }
    keep[static_cast<long long>(b) * N + p] = (p == 0 || rank >= num_drop) ? 1 : 0;
  }
}

// x[m, :] = table[src_row[m], :] (+ table[src_row2[m], :]: absolute position embeddings, open_musiclm.py:134-136);
// a negative row contributes zero.  fp32 table, fp32 out; 128-bit copies.
__global__ void embed_gather_kernel(const float* __restrict__ table, const int* __restrict__ src_row,
                                    const int* __restrict__ src_row2, float* __restrict__ x, int M, int D) {
  const int vec_per_row = D >> 2;
  const long long total = static_cast<long long>(M) * vec_per_row;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), v = static_cast<int>(i - static_cast<long long>(m) * vec_per_row);
    const int r = src_row[m];
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r >= 0) val = reinterpret_cast<const float4*>(table + static_cast<long long>(r) * D)[v];
    if (src_row2 != nullptr) {
      const int r2 = src_row2[m];
      if (r2 >= 0) {
        const float4 p = reinterpret_cast<const float4*>(table + static_cast<long long>(r2) * D)[v];
        val.x += p.x; val.y += p.y; val.z += p.z; val.w += p.w;
      }
    }
    reinterpret_cast<float4*>(x + static_cast<long long>(m) * D)[v] = val;
  }
}

// Decode step with absolute position embeddings: x[m, :] = table[src_row[m], :] + table[pos_row_base + p, :] with
// p = *pos_ptr + pos_offset, the same position row for every m (kRowPos: p = pos_ptr[m] + pos_offset, each sequence at
// its own position; kRowOffset: p = pos_ptr[m] + pos_offset_rows[m], each sequence also with its own predicted-sequence
// start, as in a generation session whose rows have conditioning of different lengths).  The position is read on the
// device, so a captured CUDA graph sees the current step on every replay.  A negative src_row, or p outside
// [0, pos_rows), contributes zero.
template <bool kRowPos, bool kRowOffset>
__device__ __forceinline__ void embed_gather_pos_body(const float* __restrict__ table, const int* __restrict__ src_row,
                                                      const int* __restrict__ pos_ptr, int pos_offset,
                                                      const int* __restrict__ pos_offset_rows, int pos_row_base, int pos_rows,
                                                      float* __restrict__ x, int M, int D) {
  const int vec_per_row = D >> 2;
  const long long total = static_cast<long long>(M) * vec_per_row;
  int p = 0;
  bool has_pos = false;
  const float4* prow = nullptr;
  if constexpr (!kRowPos) {
    p = __ldg(pos_ptr) + pos_offset;
    has_pos = p >= 0 && p < pos_rows;
    prow = reinterpret_cast<const float4*>(table + static_cast<long long>(pos_row_base + (has_pos ? p : 0)) * D);
  }
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), v = static_cast<int>(i - static_cast<long long>(m) * vec_per_row);
    if constexpr (kRowPos) {
      p = __ldg(pos_ptr + m) + (kRowOffset ? __ldg(pos_offset_rows + m) : pos_offset);
      has_pos = p >= 0 && p < pos_rows;
      prow = reinterpret_cast<const float4*>(table + static_cast<long long>(pos_row_base + (has_pos ? p : 0)) * D);
    }
    const int r = src_row[m];
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r >= 0) val = reinterpret_cast<const float4*>(table + static_cast<long long>(r) * D)[v];
    if (has_pos) {
      const float4 q = prow[v];
      val.x += q.x; val.y += q.y; val.z += q.z; val.w += q.w;
    }
    reinterpret_cast<float4*>(x + static_cast<long long>(m) * D)[v] = val;
  }
}

template <bool kRowPos>
__global__ void embed_gather_pos_kernel(const float* __restrict__ table, const int* __restrict__ src_row,
                                        const int* __restrict__ pos_ptr, int pos_offset, int pos_row_base, int pos_rows,
                                        float* __restrict__ x, int M, int D) {
  embed_gather_pos_body<kRowPos, false>(table, src_row, pos_ptr, pos_offset, nullptr, pos_row_base, pos_rows, x, M, D);
}

__global__ void embed_gather_pos_rows_kernel(const float* __restrict__ table, const int* __restrict__ src_row,
                                             const int* __restrict__ pos, const int* __restrict__ pos_offset_rows,
                                             int pos_row_base, int pos_rows, float* __restrict__ x, int M, int D) {
  embed_gather_pos_body<true, true>(table, src_row, pos, 0, pos_offset_rows, pos_row_base, pos_rows, x, M, D);
}

// dtable[src_row[m], :] += scale * dx[m, :]   (scale = grad_shrink alpha, utils.py:60-61).
__global__ void embed_scatter_kernel(float* __restrict__ dtable, const int* __restrict__ src_row,
                                     const float* __restrict__ dx, int M, int D, float scale) {
  const int vec_per_row = D >> 2;
  const long long total = static_cast<long long>(M) * vec_per_row;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), v = static_cast<int>(i - static_cast<long long>(m) * vec_per_row);
    const int r = src_row[m];
    if (r < 0) continue;
    const float4 g = reinterpret_cast<const float4*>(dx + static_cast<long long>(m) * D)[v];
    float* dst = dtable + static_cast<long long>(r) * D + v * 4;
    atomicAdd(dst + 0, g.x * scale);
    atomicAdd(dst + 1, g.y * scale);
    atomicAdd(dst + 2, g.z * scale);
    atomicAdd(dst + 3, g.w * scale);
  }
}

// Deterministic scatter-add: every destination row is summed by one warp, over its positions in ascending order.
// Pass 1 records the first position of every row (integer atomicMin: order-independent); in pass 2 the warp of that
// first position walks the remaining positions, adds the matching dx rows in order onto the table row and restores the
// row's marker to INT_MAX.  The adds are the default kernel's (dst + dx * scale, each rounded), in position order.
__global__ void embed_first_kernel(const int* __restrict__ src_row, int M, int rows, int* __restrict__ first) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int r = src_row[m];
  if (r >= 0 && r < rows) atomicMin(first + r, m);
}

template <int NCH>
__global__ void __launch_bounds__(256)
embed_scatter_det_kernel(float* __restrict__ dtable, const int* __restrict__ src_row, const float* __restrict__ dx, int M, int D,
                         int rows, float scale, int* __restrict__ first) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  const int r = src_row[m];
  if (r < 0 || r >= rows || __ldcg(first + r) != m) return;
  float* trow = dtable + static_cast<long long>(r) * D;
  float4 acc[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = (c * 32 + lane) * 4;
    acc[c] = col < D ? *reinterpret_cast<const float4*>(trow + col) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int base = m; base < M; base += 32) {
    const int idx = base + lane;
    unsigned hit = __ballot_sync(0xffffffffu, idx < M && src_row[idx] == r);
    while (hit) {
      const int mm = base + __ffs(hit) - 1;
      hit &= hit - 1;
      const float* g = dx + static_cast<long long>(mm) * D;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int col = (c * 32 + lane) * 4;
        if (col < D) {
          const float4 v = *reinterpret_cast<const float4*>(g + col);
          acc[c].x = __fadd_rn(acc[c].x, __fmul_rn(v.x, scale));
          acc[c].y = __fadd_rn(acc[c].y, __fmul_rn(v.y, scale));
          acc[c].z = __fadd_rn(acc[c].z, __fmul_rn(v.z, scale));
          acc[c].w = __fadd_rn(acc[c].w, __fmul_rn(v.w, scale));
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = (c * 32 + lane) * 4;
    if (col < D) *reinterpret_cast<float4*>(trow + col) = acc[c];
  }
  if (lane == 0) first[r] = 0x7fffffff;
}

template <int NCH>
static int launch_scatter_det(float* dtable, const int* src_row, const float* dx, int M, int D, int rows, float scale, int* first,
                              cudaStream_t st) {
  OMLM_KLAUNCH((embed_scatter_det_kernel<NCH>), (M + 7) / 8, 256, 0, st, dtable, src_row, dx, M, D, rows, scale, first);
  OMLM_LAUNCH_CHECK();
  return 0;
}

template <bool kRowPos, bool kRowOffset = false>
static int launch_embed_gather_pos(const float* table, const int* src_row, const int* pos_ptr, int pos_offset, int pos_row_base,
                                   int pos_rows, float* x, int M, int D, void* stream, const int* pos_offset_rows = nullptr) {
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0, "embed_gather_pos: bad shape %d x %d", M, D);
  OMLM_CHECK_ARG(table != nullptr && src_row != nullptr && pos_ptr != nullptr && x != nullptr &&
                 (!kRowOffset || pos_offset_rows != nullptr), "embed_gather_pos: null pointer");
  OMLM_CHECK_ARG(pos_row_base >= 0 && pos_rows > 0, "embed_gather_pos: bad position rows %d + [0, %d)", pos_row_base,
                 pos_rows);
  const long long total = static_cast<long long>(M) * (D / 4);
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(num_sms()) * 16));
  if constexpr (kRowOffset) {
    OMLM_KLAUNCH((embed_gather_pos_rows_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), table, src_row, pos_ptr,
                 pos_offset_rows, pos_row_base, pos_rows, x, M, D);
  } else {
    OMLM_KLAUNCH((embed_gather_pos_kernel<kRowPos>), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), table, src_row, pos_ptr,
                 pos_offset, pos_row_base, pos_rows, x, M, D);
  }
  OMLM_LAUNCH_CHECK();
  return 0;
}

}  // namespace omlm

extern "C" {

int omlm_token_plan(int n_seqs, const long long* const* ids, const int* len, const int* codebook,
                    const int* nq, const int* emb_row_base, const int* start_row, int B,
                    int append_eos, int drop_last, int mask_cond, int pad_id,
                    const unsigned char* mask_in, const unsigned char* forget_keep,
                    long long* ids_out, int* src_row, unsigned char* key_mask, int* labels,
                    int* err_flag, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n_seqs >= 1 && n_seqs <= OMLM_MAX_SEQS, "token_plan: n_seqs %d out of range", n_seqs);
  OMLM_CHECK_ARG(B > 0, "token_plan: empty batch");
  TokenPlanArgs a;
  a.n_seqs = n_seqs; a.append_eos = append_eos; a.drop_last = drop_last; a.mask_cond = mask_cond; a.pad_id = pad_id;
  int N = 0, n_ids = 0, n_lab = 0;
  for (int s = 0; s < n_seqs; ++s) {
    OMLM_CHECK_ARG(len[s] >= 0 && nq[s] >= 1, "token_plan: bad sequence %d", s);
    a.ids[s] = ids[s]; a.len[s] = len[s]; a.codebook[s] = codebook[s]; a.nq[s] = nq[s];
    a.emb_row_base[s] = emb_row_base[s]; a.start_row[s] = start_row[s];
    const int n_with_eos = len[s] + (append_eos ? 1 : 0);
    const int n_tok = n_with_eos - ((s == n_seqs - 1 && drop_last) ? 1 : 0);
    OMLM_CHECK_ARG(n_tok >= 0, "token_plan: sequence %d too short", s);
    N += 1 + n_tok; n_ids += n_tok; n_lab += n_with_eos;
  }
  OMLM_KLAUNCH((token_plan_kernel), B, 256, 0, reinterpret_cast<cudaStream_t>(stream), 
      a, mask_in, forget_keep, ids_out, src_row, key_mask, labels, err_flag, N, n_ids, n_lab);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_forgetful_mask(unsigned char* keep, int B, int N, int num_drop,
                        const unsigned long long* seed, unsigned long long stream_id, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && N <= 12000, "forgetful_mask: bad shape %d x %d", B, N);
  OMLM_CHECK_ARG(num_drop >= 0 && num_drop < N, "forgetful_mask: num_drop %d out of range", num_drop);
  OMLM_KLAUNCH((forgetful_mask_kernel), B, 512, N * sizeof(unsigned int), reinterpret_cast<cudaStream_t>(stream), 
      keep, N, num_drop, seed, stream_id);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_embed_gather(const float* table, const int* src_row, const int* src_row2, float* x, int M, int D, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0, "embed_gather: bad shape %d x %d", M, D);
  const long long total = static_cast<long long>(M) * (D / 4);
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(num_sms()) * 16));
  OMLM_KLAUNCH((embed_gather_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), table, src_row, src_row2, x, M, D);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_embed_gather_pos(const float* table, const int* src_row, const int* pos_ptr, int pos_offset, int pos_row_base,
                          int pos_rows, float* x, int M, int D, void* stream) {
  return omlm::launch_embed_gather_pos<false>(table, src_row, pos_ptr, pos_offset, pos_row_base, pos_rows, x, M, D, stream);
}

int omlm_embed_gather_pos_ragged(const float* table, const int* src_row, const int* pos, int pos_offset, int pos_row_base,
                                 int pos_rows, float* x, int M, int D, void* stream) {
  return omlm::launch_embed_gather_pos<true>(table, src_row, pos, pos_offset, pos_row_base, pos_rows, x, M, D, stream);
}

int omlm_embed_gather_pos_rows(const float* table, const int* src_row, const int* pos, const int* pos_offset, int pos_row_base,
                               int pos_rows, float* x, int M, int D, void* stream) {
  return omlm::launch_embed_gather_pos<true, true>(table, src_row, pos, 0, pos_row_base, pos_rows, x, M, D, stream, pos_offset);
}

int omlm_embed_scatter_add(float* dtable, const int* src_row, const float* dx, int M, int D,
                           float scale, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0, "embed_scatter: bad shape %d x %d", M, D);
  const long long total = static_cast<long long>(M) * (D / 4);
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(num_sms()) * 16));
  OMLM_KLAUNCH((embed_scatter_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), dtable, src_row, dx, M, D, scale);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_embed_scatter_add_det(float* dtable, const int* src_row, const float* dx, int M, int D, float scale, int* first_ws,
                               int table_rows, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "embed_scatter_det: bad shape %d x %d", M, D);
  OMLM_CHECK_ARG(first_ws != nullptr && table_rows > 0, "embed_scatter_det: no row-marker workspace");
  auto st = reinterpret_cast<cudaStream_t>(stream);
  OMLM_KLAUNCH((embed_first_kernel), (M + 255) / 256, 256, 0, st, src_row, M, table_rows, first_ws);
  OMLM_LAUNCH_CHECK();
  const int nch = (D + 127) / 128;
  if (nch <= 1) return launch_scatter_det<1>(dtable, src_row, dx, M, D, table_rows, scale, first_ws, st);
  if (nch <= 2) return launch_scatter_det<2>(dtable, src_row, dx, M, D, table_rows, scale, first_ws, st);
  if (nch <= 4) return launch_scatter_det<4>(dtable, src_row, dx, M, D, table_rows, scale, first_ws, st);
  if (nch <= 8) return launch_scatter_det<8>(dtable, src_row, dx, M, D, table_rows, scale, first_ws, st);
  return launch_scatter_det<16>(dtable, src_row, dx, M, D, table_rows, scale, first_ws, st);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ token store
// Batch assembly from a device-resident token store (the pre-tokenised dataset of open_musiclm/data.py:304-438 kept in
// HBM as flat int16 arrays): out[b, t, c] = (long) src[(start[b] + t) * width + c] for t < len, c < width.  One random
// crop per batch row; the crop indices are drawn on the host with the reference's arithmetic, the copy never leaves HBM.
namespace omlm {
__global__ void gather_windows_kernel(const short* __restrict__ src, const long long* __restrict__ start, long long* __restrict__ out,
                                      int len, int width, int B) {
  const long long per_row = static_cast<long long>(len) * width;
  const long long total = per_row * B;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per_row);
    const long long r = i - b * per_row;
    out[i] = static_cast<unsigned short>(src[start[b] * width + r]);
  }
}
}  // namespace omlm

extern "C" int omlm_gather_windows(const void* src_i16, const long long* start, long long* out, int len, int width, int B, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && len >= 0 && width > 0, "gather_windows: bad shape");
  if (len == 0) return 0;
  const long long total = static_cast<long long>(len) * width * B;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(num_sms()) * 8));
  OMLM_KLAUNCH((gather_windows_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const short*>(src_i16), start, out, len, width, B);
  OMLM_LAUNCH_CHECK();
  return 0;
}
