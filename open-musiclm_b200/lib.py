"""ctypes binding of libomlm_b200.so (the C ABI declared in include/omlm_b200.h).

There is no fallback: if the shared library is missing or a call fails, this module raises.
PyTorch is used only for device memory and streams; every tensor is passed as a raw pointer.
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libomlm_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "omlm_b200.h")

_lib = None


class OmlmError(RuntimeError):
    pass


def header_symbols():
    """Every function name declared in include/omlm_b200.h."""
    with open(HEADER_PATH) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(omlm_[a-z0-9_]+)\s*\(", src)))


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OmlmError(
                f"{LIB_PATH} not found - build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU or PyTorch fallback for the hot path)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.omlm_last_error.restype = ctypes.c_char_p
    return _lib


def _check(rc, name):
    if rc != 0:
        msg = load().omlm_last_error().decode(errors="replace")
        raise OmlmError(f"{name} failed (rc={rc}): {msg}")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


_I = ctypes.c_int
_L = ctypes.c_long
_F = ctypes.c_float


def call(name, *args):
    """Call an int-returning entry point; raise with omlm_last_error() on failure."""
    fn = getattr(load(), name)
    rc = fn(*args)
    _check(rc, name)


_T16 = (torch.bfloat16, torch.float16)
FMT = {torch.bfloat16: 0, torch.float32: 1, torch.float16: 2}      # kFmtBF16 / kFmtF32 / kFmtF16 (csrc/common.cuh)


def device_check():
    call("omlm_device_check")


def num_sms():
    return int(load().omlm_num_sms())


def gemm(a, b, out, *, a_mn=False, b_mn=False, M=None, N=None, K=None, addend=None, alpha=1.0,
         splits=1, row_split=0, row_valid=0, n_valid=0, block_n=128, max_ctas=0):
    """out[m,n] = alpha * sum_k A(m,k) B(n,k) (+ addend).  a: [M,K] (or [K,M] if a_mn); b: [N,K] (or [K,N] if b_mn).
    Each operand is bf16 or fp16 (its torch dtype decides the tensor-core operand format), fp32 accumulation."""
    assert a.dtype in _T16 and b.dtype in _T16
    assert a.stride(-1) == 1 and b.stride(-1) == 1 and out.stride(-1) == 1
    if M is None:
        M = a.shape[1] if a_mn else a.shape[0]
    if K is None:
        K = a.shape[0] if a_mn else a.shape[1]
    if N is None:
        N = b.shape[1] if b_mn else b.shape[0]
    out_f32 = 1 if out.dtype == torch.float32 else 0
    assert out_f32 or out.dtype == torch.bfloat16
    call("omlm_gemm16", _p(a), _I(int(a.dtype == torch.float16)), _I(int(a_mn)), _L(a.stride(0)),
         _p(b), _I(int(b.dtype == torch.float16)), _I(int(b_mn)), _L(b.stride(0)),
         _I(M), _I(N), _I(K), _p(out), _I(out_f32), _L(out.stride(0)),
         _p(addend), _L(addend.stride(0) if addend is not None else 0), _F(alpha), _I(splits),
         _I(row_split), _I(row_valid), _I(n_valid), _I(block_n), _I(max_ctas), _stream())
    return out


# ------------------------------------------------------------------------------------------------
# thin tensor-level wrappers (tensors in, raw pointers out); shapes are validated on the C side
# ------------------------------------------------------------------------------------------------
_ULL = ctypes.c_ulonglong


def token_plan(ids_list, codebooks, nqs, emb_row_base, start_row, *, append_eos, drop_last, mask_cond,
               pad_id=-1, mask_in=None, forget_keep=None, want_labels=True, err_flag=None):
    """Returns ids_out [B, sum n_tok] int64, src_row [B,N] int32, key_mask [B,N] uint8, labels [B, sum(len+eos)] int32."""
    S = len(ids_list)
    B = ids_list[0].shape[0]
    dev = ids_list[0].device
    flat = [t.reshape(B, -1).contiguous() for t in ids_list]
    assert all(t.dtype == torch.int64 for t in flat)
    lens = [t.shape[1] for t in flat]
    n_tok = [l + (1 if append_eos else 0) - (1 if (drop_last and s == S - 1) else 0) for s, l in enumerate(lens)]
    N = sum(n + 1 for n in n_tok)
    ids_out = torch.empty(B, sum(n_tok), dtype=torch.int64, device=dev)
    src_row = torch.empty(B, N, dtype=torch.int32, device=dev)
    key_mask = torch.empty(B, N, dtype=torch.uint8, device=dev)
    n_lab = sum(l + (1 if append_eos else 0) for l in lens)
    labels = torch.empty(B, n_lab, dtype=torch.int32, device=dev) if want_labels else None
    ptrs = (ctypes.c_void_p * S)(*[t.data_ptr() for t in flat])
    arr = lambda v: (ctypes.c_int * S)(*[int(x) for x in v])
    call("omlm_token_plan", _I(S), ptrs, arr(lens), arr(codebooks), arr(nqs), arr(emb_row_base), arr(start_row),
         _I(B), _I(int(append_eos)), _I(int(drop_last)), _I(int(mask_cond)), _I(pad_id), _p(mask_in), _p(forget_keep),
         _p(ids_out), _p(src_row), _p(key_mask), _p(labels), _p(err_flag), _stream())
    return ids_out, src_row, key_mask, labels, n_tok


def forgetful_mask(B, N, num_drop, seed_tensor, stream_id, device):
    keep = torch.empty(B, N, dtype=torch.uint8, device=device)
    call("omlm_forgetful_mask", _p(keep), _I(B), _I(N), _I(num_drop), _p(seed_tensor), _ULL(stream_id), _stream())
    return keep


def embed_gather(table, src_row, x, src_row2=None):
    """x[m] = table[src_row[m]] (+ table[src_row2[m]]); negative rows contribute zero."""
    M, D = x.shape
    call("omlm_embed_gather", _p(table), _p(src_row), _p(src_row2), _p(x), _I(M), _I(D), _stream())


def embed_scatter_add(dtable, src_row, dx, scale):
    M, D = dx.shape
    call("omlm_embed_scatter_add", _p(dtable), _p(src_row), _p(dx), _I(M), _I(D), _F(scale), _stream())


def layernorm_fwd(x, gamma, y, xraw=None, stats=None, dest_row=None, ycopy=None):
    """y: fp16 or bf16 (its dtype decides); ycopy: optional bf16 duplicate of y for the backward GEMMs."""
    M, D = x.shape
    assert y.dtype in _T16 and (xraw is None or xraw.dtype == torch.bfloat16) and (ycopy is None or ycopy.dtype == torch.bfloat16)
    call("omlm_layernorm_fwd", _p(x), _p(gamma), _p(y), _I(int(y.dtype == torch.float16)), _p(ycopy), _p(xraw), _p(stats),
         _p(dest_row), _I(M), _I(D), _stream())


def layernorm_bwd(dy, x, stats, gamma, dx, dgamma, dres=None, draw=None, src_row=None, dx_bf16=None):
    M, D = x.shape
    call("omlm_layernorm_bwd", _p(dy), _p(x), _p(stats), _p(gamma), _p(dres), _p(draw), _p(src_row), _p(dx),
         _p(dx_bf16), _p(dgamma), _I(M), _I(D), _stream())


def qk_l2norm_fwd(q_raw, kv_raw, q_scale, k_scale, qn, kvn, heads):
    call("omlm_qk_l2norm_fwd", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(qn), _p(kvn),
         _I(q_raw.shape[0]), _I(heads), _stream())


def qk_l2norm_bwd(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, heads):
    call("omlm_qk_l2norm_bwd", _p(dqn), _p(dkvn), _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(dq_raw),
         _p(dkv_raw), _p(dq_scale), _p(dk_scale), _I(q_raw.shape[0]), _I(heads), _stream())


def sgemm_small(A, sa, B, sb, C, sc, M, N, K, *, Z=None, bias=None, act=0, accumulate=False):
    call("omlm_sgemm_small", _p(A), _L(sa[0]), _L(sa[1]), _p(B), _L(sb[0]), _L(sb[1]), _p(C), _L(sc[0]), _L(sc[1]),
         _p(Z), _p(bias), _I(M), _I(N), _I(K), _I(act), _I(int(accumulate)), _stream())


def silu_bwd(dA, Z, dZ, dZ_bf16=None):
    call("omlm_silu_bwd", _p(dA), _p(Z), _p(dZ), _p(dZ_bf16), _L(dA.numel()), _stream())


def split3_bf16(src, dst, weight_mode=False):
    R, C = src.shape
    call("omlm_split3_bf16", _p(src), _L(src.stride(0)), _p(dst), _I(R), _I(C), _I(int(weight_mode)), _stream())


def bias_silu(z, bias, a):
    R, C = z.shape
    call("omlm_bias_silu", _p(z), _p(bias), _p(a), _I(R), _I(C), _stream())


def colsum(X, s_m, s_n, out, M, N, accumulate=False):
    call("omlm_colsum", _p(X), _L(s_m), _L(s_n), _p(out), _I(M), _I(N), _I(int(accumulate)), _stream())


def arange_f32(out):
    call("omlm_arange_f32", _p(out), _I(out.numel()), _stream())


def attn_fwd(qn, kvn, table, key_mask, out, lse2, B, N, heads, scale=8.0):
    call("omlm_attn_fwd", _p(qn), _p(kvn), _p(table), _I(table.stride(0)), _p(key_mask), _p(out), _p(lse2),
         _I(B), _I(N), _I(heads), _F(scale), _stream())


def attn_fwd_tc(qn, kvn, table, key_mask, out, lse2, B, N, heads, scale=8.0):
    call("omlm_attn_fwd_tc", _p(qn), _p(kvn), _p(table), _I(table.stride(0)), _p(key_mask), _p(out), _p(lse2),
         _I(B), _I(N), _I(heads), _F(scale), _stream())


def attn_bwd(qn, kvn, d_o, o, lse2, table, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads, scale=8.0):
    call("omlm_attn_bwd", _p(qn), _p(kvn), _p(d_o), _p(o), _p(lse2), _p(table), _I(table.stride(0)), _p(key_mask),
         _p(dsum_scratch), _p(dqn), _p(dkvn), _p(dtable), _I(B), _I(N), _I(heads), _F(scale), _stream())


def attn_bwd_tc(qn, kvn, d_o, o, lse2, table, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads, scale=8.0):
    call("omlm_attn_bwd_tc", _p(qn), _p(kvn), _p(d_o), _p(o), _p(lse2), _p(table), _I(table.stride(0)), _p(key_mask),
         _p(dsum_scratch), _p(dqn), _p(dkvn), _p(dtable), _I(B), _I(N), _I(heads), _F(scale), _stream())


def gemm_ffn_up(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, Nseq, Fp, max_ctas=0):
    M, K = xn.shape
    assert xn.dtype in _T16 and xn.dtype == w1_packed.dtype == u_out.dtype == h_out.dtype
    call("omlm_gemm_ffn_up", _p(xn), _p(w1_packed), _p(conv_w_packed), _p(u_out), _p(h_out), _p(rowsum), _I(M), _I(Nseq),
         _I(K), _I(Fp), _I(int(xn.dtype == torch.float16)), _I(max_ctas), _stream())


def ffn_norm_fwd(h, rowsum, gamma, hn, stats, F, Fp, drop_p=0.0, seed=None, layer=0, keep_bits=None, hn_copy=None):
    assert h.dtype in _T16 and h.dtype == hn.dtype and (hn_copy is None or hn_copy.dtype == torch.bfloat16)
    call("omlm_ffn_norm_fwd", _p(h), _p(rowsum), _p(gamma), _p(hn), _p(hn_copy), _p(stats), _p(keep_bits), _L(h.shape[0]),
         _I(F), _I(Fp), _F(drop_p), _p(seed), _I(layer), _I(int(h.dtype == torch.float16)), _stream())


def ffn_mid_bwd(dhn, hn, u, stats, conv_w, gamma, rowstat, du, dgamma, dconv_w, B, N, F, Fp, drop_p=0.0, keep_bits=None, rowstat_parts=0):
    """dgamma [F] / dconv_w [2F, 3] (or None) are accumulated in the parameters' own layouts; rowstat_parts > 0: rowstat
    holds the partial row sums written by gemm_rowstat, else it is a [M, 2] scratch."""
    assert u.dtype in _T16 and hn.dtype == dhn.dtype == du.dtype == torch.bfloat16
    assert dgamma.numel() == F and (dconv_w is None or dconv_w.numel() == 6 * F)
    call("omlm_ffn_mid_bwd", _p(dhn), _p(hn), _p(u), _p(stats), _p(conv_w), _p(gamma), _p(keep_bits), _p(rowstat), _I(rowstat_parts), _p(du),
         _p(dgamma), _p(dconv_w), _I(B), _I(N), _I(F), _I(Fp), _F(drop_p), _I(int(u.dtype == torch.float16)), _stream())


def gemm_rowstat(a, b, out, hn, gamma, part, *, b_mn=False, M=None, N=None, K=None, keep_bits=None, keep_scale=1.0, max_ctas=0):
    """out = a b^T (dense bf16 [M, N], 256-wide tiles) + per-row partial sums against hn in the epilogue (omlm_gemm16_rowstat)."""
    assert a.dtype in _T16 and b.dtype == a.dtype and out.dtype == hn.dtype == torch.bfloat16 and part.dtype == torch.float32
    M = a.shape[0] if M is None else M
    K = a.shape[1] if K is None else K
    N = (b.shape[1] if b_mn else b.shape[0]) if N is None else N
    assert part.numel() == M * (N // 128) * 2
    call("omlm_gemm16_rowstat", _p(a), _I(int(a.dtype == torch.float16)), _I(0), _L(a.stride(0)), _p(b), _I(int(b.dtype == torch.float16)),
         _I(int(b_mn)), _L(b.stride(0)), _I(M), _I(N), _I(K), _p(out), _L(out.stride(0)), _p(hn), _L(hn.stride(0)), _p(keep_bits), _p(gamma),
         _F(keep_scale), _p(part), _I(N // 128), _I(max_ctas), _stream())
    return out


def cross_entropy(logits, labels, C, loss_acc, *, grad_scale=0.0, dlogits=None, ignore_index=-100, label_stride=1, rows=None,
                  rows_per_batch=0, batch_stride=0, loss_scale=1.0):
    """labels: int32; flat (rows_per_batch = 0) or the strided view described in include/omlm_b200.h (pass the tensor whose
    data_ptr is the first label of the group)."""
    rows = logits.shape[0] if rows is None else rows
    call("omlm_cross_entropy", _p(logits), _L(logits.stride(0)), _p(labels), _I(label_stride), _I(rows_per_batch), _L(batch_stride),
         _I(rows), _I(C), _I(ignore_index), _F(grad_scale), _F(loss_scale), _p(dlogits),
         _L(dlogits.stride(0) if dlogits is not None else 0), _I(dlogits.shape[1] if dlogits is not None else 0), _p(loss_acc), _stream())


def grad_sumsq(g, acc, prescale=1.0):
    call("omlm_grad_sumsq", _p(g), _L(g.numel()), _F(prescale), _p(acc), _stream())


def adamw_step(p, g, m, v, n_decay, hyper, sumsq):
    call("omlm_adamw_step", _p(p), _p(g), _p(m), _p(v), _L(p.numel()), _L(n_decay), _p(hyper), _p(sumsq), _stream())


def pack(src, src_ld, rows_valid, cols_valid, dst, rows_p, cols_p, split_dst=0, split_src=0):
    call("omlm_pack", _p(src), _L(src_ld), _I(rows_valid), _I(cols_valid), _p(dst), _I(FMT[dst.dtype]),
         _L(cols_p if dst.dim() == 1 else dst.stride(0)), _I(rows_p), _I(cols_p), _I(split_dst), _I(split_src), _stream())


class _PackJob(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("dst", ctypes.c_void_p), ("dst2", ctypes.c_void_p), ("src_ld", ctypes.c_long),
                ("dst_ld", ctypes.c_long), ("unit_start", ctypes.c_long), ("rows_valid", ctypes.c_int), ("cols_valid", ctypes.c_int),
                ("rows_p", ctypes.c_int), ("cols_p", ctypes.c_int), ("split_dst", ctypes.c_int), ("split_src", ctypes.c_int),
                ("dst_fmt", ctypes.c_int), ("dst2_fmt", ctypes.c_int)]


class PackTable:
    """Device-resident table of pack jobs (same arguments as pack()); run() repacks all of them in one launch per
    MAX_JOBS jobs (a 24-layer model has ~170 jobs: one launch)."""
    MAX_JOBS = 512      # kPackMaxJobs in csrc/optim.cu

    def __init__(self, device):
        self.device, self.chunks, self.keep, self.tables = device, [[[], 0]], [], None

    UNIT = 1024         # quads (4 consecutive columns of a destination row) per work unit: kPackUnit in csrc/optim.cu

    def add(self, src, src_ld, rows_valid, cols_valid, dst, rows_p, cols_p, split_dst=0, split_src=0, dst2=None):
        """dst2: optional second destination with dst's geometry (another 16-bit format), written from the same read."""
        if len(self.chunks[-1][0]) == self.MAX_JOBS:
            self.chunks.append([[], 0])
        chunk = self.chunks[-1]
        dst_ld = cols_p if dst.dim() == 1 else dst.stride(0)
        if dst2 is not None:
            assert dst2.shape == dst.shape and dst2.stride() == dst.stride() and dst2.element_size() == dst.element_size()
        chunk[0].append(_PackJob(src.data_ptr(), dst.data_ptr(), dst2.data_ptr() if dst2 is not None else None, src_ld, dst_ld, chunk[1],
                                 rows_valid, cols_valid, rows_p, cols_p, split_dst, split_src, FMT[dst.dtype],
                                 FMT[dst2.dtype] if dst2 is not None else 0))
        self.keep.append((src, dst, dst2))
        chunk[1] += (rows_p * ((cols_p + 3) // 4) + self.UNIT - 1) // self.UNIT
        self.tables = None

    @property
    def n_jobs(self):
        return sum(len(c[0]) for c in self.chunks)

    def run(self):
        if self.tables is None:
            self.tables = []
            for jobs, units in self.chunks:
                arr = (_PackJob * len(jobs))(*jobs)
                host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
                self.tables.append((host.to(self.device), len(jobs), units))
        for table, n, units in self.tables:
            call("omlm_pack_multi", ctypes.c_void_p(table.data_ptr()), _I(n), _L(units), _stream())


def unpack_add(packed, rows_p, cols_p, dst, dst_ld, rows_valid, cols_valid, split_dst=0, split_src=0):
    call("omlm_unpack_add", _p(packed), _L(cols_p if packed.dim() == 1 else packed.stride(0)), _I(rows_p), _I(cols_p),
         _p(dst), _L(dst_ld), _I(rows_valid), _I(cols_valid), _I(split_dst), _I(split_src), _stream())


# ------------------------------------------------------------------------------------------------ incremental decoding
def skinny_gemm(A, W, out, *, prologue=0, gamma=None, rowsum=None, n_real=0, addend=None):
    """out[b, n] = A[b, :] . W[n, :] (+ addend) for B <= 16 rows; prologue: see include/omlm_b200.h."""
    B = A.shape[0]
    N, K = W.shape
    assert W.dtype in _T16 and W.stride(1) == 1 and out.stride(-1) == 1 and A.stride(-1) == 1
    assert (prologue in (0, 3) and A.dtype == W.dtype) or (prologue in (1, 2) and A.dtype == torch.float32)
    call("omlm_skinny_gemm", _p(A), _L(A.stride(0)), _I(prologue), _p(W), _L(W.stride(0)), _I(int(W.dtype == torch.float16)),
         _p(gamma), _p(rowsum), _I(n_real), _p(addend), _L(addend.stride(0) if addend is not None else 0), _p(out),
         _I(FMT[out.dtype]), _L(out.stride(0)), _I(B), _I(N), _I(K), _stream())


def decode_gemm_workspace(B, N, K):
    """Bytes of split-K partials omlm_decode_gemm needs for a B x N x K call on the current device."""
    part = _L(0)
    call("omlm_decode_gemm_workspace", _I(B), _I(N), _I(K), ctypes.byref(part))
    return part.value


class DecodeWorkspace:
    """Scratch of the large-batch decode kernels, allocated once so that CUDA-graph capture allocates nothing:
    the 16-bit activation operand [B, max K], the split-K partials, the attention's per-slice partials and its
    per-sequence counters (zero; every call leaves them zero).  shapes: the (N, K) of every decode_gemm call; max_pos /
    heads: attention."""

    def __init__(self, device, B, shapes, max_pos=0, heads=0):
        part = max(decode_gemm_workspace(B, N, K) for N, K in shapes)
        attn = B * -(-max_pos // 128) * heads * 66 if max_pos else 0
        self.a16 = torch.empty(B * max(K for _, K in shapes), device=device, dtype=torch.int16)
        self.part = torch.empty(max(part // 4, 1), device=device, dtype=torch.float32)
        self.attn = torch.empty(max(attn, 1), device=device, dtype=torch.float32)
        self.counters = torch.zeros(B, device=device, dtype=torch.int32)


def decode_gemm(A, W, out, *, prologue=0, gamma=None, rowsum=None, n_real=0, addend=None, ws=None):
    """skinny_gemm's contract for 1 <= B <= 256 rows on the tensor cores (omlm_decode_gemm).  ws: a DecodeWorkspace
    covering this shape (None: a fresh one, which is not CUDA-graph capturable)."""
    B = A.shape[0]
    N, K = W.shape
    assert W.dtype in _T16 and W.stride(1) == 1 and out.stride(-1) == 1 and A.stride(-1) == 1
    assert (prologue in (0, 3) and A.dtype == W.dtype) or (prologue in (1, 2) and A.dtype == torch.float32)
    if ws is None:
        ws = DecodeWorkspace(A.device, B, [(N, K)])
    call("omlm_decode_gemm", _p(A), _L(A.stride(0)), _I(prologue), _p(W), _L(W.stride(0)), _I(int(W.dtype == torch.float16)),
         _p(gamma), _p(rowsum), _I(n_real), _p(addend), _L(addend.stride(0) if addend is not None else 0), _p(out),
         _I(FMT[out.dtype]), _L(out.stride(0)), _I(B), _I(N), _I(K), _p(ws.a16), _p(ws.part), _L(ws.part.numel() * 4),
         _stream())


def attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, ws=None, scale=8.0):
    """attn_decode's contract with every cached row read once per sequence (omlm_attn_decode_mqa), 1 <= heads <= 16."""
    B = q_raw.shape[0]
    if ws is None:
        ws = DecodeWorkspace(q_raw.device, B, [(1, 8)], max_pos=max_pos, heads=heads)
    call("omlm_attn_decode_mqa", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(cache), _L(cache.stride(0)), _p(table),
         _I(table.stride(0)), _p(pos), _I(max_pos), _p(out), _I(B), _I(heads), _F(scale), _p(ws.attn), _L(ws.attn.numel() * 4),
         _p(ws.counters), _stream())


class _DecodeLayer(ctypes.Structure):
    """omlm_decode_layer (include/omlm_b200.h): the per-layer pointers of the fused decode step."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("wq", "wkv", "wo", "w1", "w2", "conv", "gin", "g_attn", "g_ff", "q_scale", "k_scale",
                                                "cache", "conv_state")]


def decode_layer_table(layers, device):
    """layers: list of dicts of tensors keyed like _DecodeLayer's fields -> (device table, keep-alive list)."""
    arr = (_DecodeLayer * len(layers))(*[_DecodeLayer(*[ly[n].data_ptr() for n, _ in _DecodeLayer._fields_]) for ly in layers])
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host.to(device), [t for ly in layers for t in ly.values()]


def decode_step(table_dev, L, B, d, heads, F, Fp, n_max, act_f16, emb_table, next_row, bias_table, pos, x0, x1, q_raw, kv_raw, o,
                hbuf, hf32, w_logit, g_final, logits, barrier, err_flag, scale=8.0):
    call("omlm_decode_step", ctypes.c_void_p(table_dev.data_ptr()), _I(L), _I(B), _I(d), _I(heads), _I(F), _I(Fp), _I(n_max), _I(int(act_f16)),
         _p(emb_table), _p(next_row), _p(bias_table), _I(bias_table.stride(0)), _p(pos), _p(x0), _p(x1), _p(q_raw), _p(kv_raw), _p(o),
         _p(hbuf), _p(hf32), _p(w_logit), _I(w_logit.shape[0]), _p(g_final), _p(logits), _L(logits.stride(0)), _p(barrier), _p(err_flag),
         _F(scale), _stream())


def attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, scale=8.0):
    call("omlm_attn_decode", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(cache), _L(cache.stride(0)), _p(table),
         _I(table.stride(0)), _p(pos), _I(max_pos), _p(out), _I(q_raw.shape[0]), _I(heads), _F(scale), _stream())


def decode_conv_geglu(u_new, state, conv_w, h_out, rowsum):
    B, Fp2 = u_new.shape
    assert u_new.dtype == state.dtype == h_out.dtype and u_new.dtype in _T16
    call("omlm_decode_conv_geglu", _p(u_new), _p(state), _p(conv_w), _p(h_out), _p(rowsum), _I(B), _I(Fp2 // 2),
         _I(int(u_new.dtype == torch.float16)), _stream())


def sample(logits, C, top_k, temperature, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B):
    call("omlm_sample", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _F(temperature), _I(int(allow_eos)), _p(uniform),
         _p(seed), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(counters), _p(pos), _I(B), _stream())


def gather_windows(src_i16, start, out):
    """out[b, t, c] = src[(start[b] + t), c] for a flat [T_total, width] int16 token store (ids are uint16)."""
    B, length = out.shape[0], out.shape[1]
    width = src_i16.shape[1] if src_i16.dim() == 2 else 1
    assert src_i16.dtype == torch.int16 and start.dtype == torch.int64 and out.dtype == torch.int64 and out.is_contiguous()
    call("omlm_gather_windows", _p(src_i16), _p(start), _p(out), _I(length), _I(width), _I(B), _stream())
