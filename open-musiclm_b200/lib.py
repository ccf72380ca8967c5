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


def gemm_splitk_det_workspace(M, N, K, splits, row_split=0, row_valid=0, n_valid=0):
    """Bytes of fp32 partials gemm_splitk_det needs (0 when the clamped split count is 1)."""
    out = _L(0)
    call("omlm_gemm16_splitk_det_workspace", _I(M), _I(N), _I(K), _I(splits), _I(row_split), _I(row_valid), _I(n_valid), ctypes.byref(out))
    return out.value


def gemm_splitk_det(a, b, out, part, *, a_mn=False, b_mn=False, M, N, K, splits, row_split=0, row_valid=0, n_valid=0,
                    block_n=128, max_ctas=0):
    """out (fp32) += A B with split-K partials summed in split order (omlm_gemm16_splitk_det); part: fp32 scratch."""
    assert a.dtype in _T16 and b.dtype in _T16 and out.dtype == torch.float32 and part.dtype == torch.float32
    call("omlm_gemm16_splitk_det", _p(a), _I(int(a.dtype == torch.float16)), _I(int(a_mn)), _L(a.stride(0)),
         _p(b), _I(int(b.dtype == torch.float16)), _I(int(b_mn)), _L(b.stride(0)), _I(M), _I(N), _I(K), _p(out), _L(out.stride(0)),
         _I(splits), _I(row_split), _I(row_valid), _I(n_valid), _I(block_n), _I(max_ctas), _p(part), _L(part.numel() * 4), _stream())
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


def embed_gather_pos(table, src_row, pos, pos_offset, pos_row_base, pos_rows, x, ragged=False):
    """x[m] = table[src_row[m]] + table[pos_row_base + pos[0] + pos_offset]; pos: int32 device tensor read by the
    kernel (so a captured graph uses its current value).  A position outside [0, pos_rows) adds nothing.
    ragged: pos holds one position per row, pos[m] (omlm_embed_gather_pos_ragged)."""
    assert pos.dtype == torch.int32 and pos.is_cuda
    M, D = x.shape
    if ragged:
        _check_row_pos(pos, M)
    call("omlm_embed_gather_pos_ragged" if ragged else "omlm_embed_gather_pos", _p(table), _p(src_row), _p(pos), _I(pos_offset),
         _I(pos_row_base), _I(pos_rows), _p(x), _I(M), _I(D), _stream())


def embed_gather_pos_rows(table, src_row, pos, pos_offset, pos_row_base, pos_rows, x):
    """embed_gather_pos with a position and a predicted-sequence offset per row: x[m] = table[src_row[m]] +
    table[pos_row_base + pos[m] + pos_offset[m]] (int32 device tensors [M]; omlm_embed_gather_pos_rows)."""
    M, D = x.shape
    _check_row_pos(pos, M)
    _check_row_pos(pos_offset, M)
    call("omlm_embed_gather_pos_rows", _p(table), _p(src_row), _p(pos), _p(pos_offset), _I(pos_row_base), _I(pos_rows), _p(x),
         _I(M), _I(D), _stream())


def embed_scatter_add(dtable, src_row, dx, scale, first=None):
    """first: int32 row markers (INT_MAX, one per table row) -> the deterministic variant (omlm_embed_scatter_add_det)."""
    M, D = dx.shape
    if first is None:
        call("omlm_embed_scatter_add", _p(dtable), _p(src_row), _p(dx), _I(M), _I(D), _F(scale), _stream())
    else:
        call("omlm_embed_scatter_add_det", _p(dtable), _p(src_row), _p(dx), _I(M), _I(D), _F(scale), _p(first),
             _I(first.numel()), _stream())


def embed_row_markers(rows, device):
    """The row markers embed_scatter_add's deterministic variant needs (every call leaves them as made here)."""
    return torch.full((rows,), 0x7FFFFFFF, dtype=torch.int32, device=device)


def layernorm_fwd(x, gamma, y, xraw=None, stats=None, dest_row=None, ycopy=None):
    """y: fp16 or bf16 (its dtype decides); ycopy: optional bf16 duplicate of y for the backward GEMMs."""
    M, D = x.shape
    assert y.dtype in _T16 and (xraw is None or xraw.dtype == torch.bfloat16) and (ycopy is None or ycopy.dtype == torch.bfloat16)
    call("omlm_layernorm_fwd", _p(x), _p(gamma), _p(y), _I(int(y.dtype == torch.float16)), _p(ycopy), _p(xraw), _p(stats),
         _p(dest_row), _I(M), _I(D), _stream())


def layernorm_bwd(dy, x, stats, gamma, dx, dgamma, dres=None, draw=None, src_row=None, dx_bf16=None, part=None):
    """part: fp32 scratch -> the deterministic variant (omlm_layernorm_bwd_det)."""
    M, D = x.shape
    args = (_p(dy), _p(x), _p(stats), _p(gamma), _p(dres), _p(draw), _p(src_row), _p(dx), _p(dx_bf16), _p(dgamma), _I(M), _I(D))
    if part is None:
        call("omlm_layernorm_bwd", *args, _stream())
    else:
        call("omlm_layernorm_bwd_det", *args, _p(part), _L(part.numel() * 4), _stream())


def qk_l2norm_fwd(q_raw, kv_raw, q_scale, k_scale, qn, kvn, heads):
    call("omlm_qk_l2norm_fwd", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(qn), _p(kvn),
         _I(q_raw.shape[0]), _I(heads), _stream())


def qk_l2norm_bwd(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, heads, part=None):
    args = (_p(dqn), _p(dkvn), _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(dq_raw), _p(dkv_raw), _p(dq_scale), _p(dk_scale),
            _I(q_raw.shape[0]), _I(heads))
    if part is None:
        call("omlm_qk_l2norm_bwd", *args, _stream())
    else:
        call("omlm_qk_l2norm_bwd_det", *args, _p(part), _L(part.numel() * 4), _stream())


def sgemm_small(A, sa, B, sb, C, sc, M, N, K, *, Z=None, bias=None, act=0, accumulate=False, det=False):
    call("omlm_sgemm_small_det" if det else "omlm_sgemm_small", _p(A), _L(sa[0]), _L(sa[1]), _p(B), _L(sb[0]), _L(sb[1]), _p(C), _L(sc[0]), _L(sc[1]),
         _p(Z), _p(bias), _I(M), _I(N), _I(K), _I(act), _I(int(accumulate)), _stream())


def silu_bwd(dA, Z, dZ, dZ_bf16=None):
    call("omlm_silu_bwd", _p(dA), _p(Z), _p(dZ), _p(dZ_bf16), _L(dA.numel()), _stream())


def split3_bf16(src, dst, weight_mode=False):
    """dst bf16 [R, 3 Cpad] (contiguous) = the three split thirds of src [R, C], each Cpad = dst.shape[1] / 3 wide."""
    R, C = src.shape
    assert dst.dtype == torch.bfloat16 and dst.is_contiguous() and dst.shape[0] == R and dst.shape[1] % 3 == 0
    call("omlm_split3_bf16", _p(src), _L(src.stride(0)), _p(dst), _I(R), _I(C), _I(dst.shape[1] // 3), _I(int(weight_mode)),
         _stream())


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


def attn_fwd_tc_varlen(qn, kvn, table, work, seq_start, seq_len, max_len, out, lse2, heads, scale=8.0):
    """attn_fwd_tc over packed sequences (omlm_attn_fwd_tc_varlen): qn [M, heads*64], kvn [M, 128]; work int32 [n_work, 2]
    of (sequence, row block) pairs; seq_start, seq_len int32 [n_seq]; max_len >= every seq_len."""
    for t in (work, seq_start, seq_len):
        assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous()
    call("omlm_attn_fwd_tc_varlen", _p(qn), _p(kvn), _p(table), _I(table.stride(0)), _p(work), _I(work.numel() // 2), _p(seq_start),
         _p(seq_len), _I(qn.shape[0]), _I(max_len), _p(out), _p(lse2), _I(heads), _F(scale), _stream())


def attn_fwd_tc_chunk(qn, kv, table, work, seq_start, seq_len, q_off, kv_start, max_end, out, lse2, heads, scale=8.0):
    """attn_fwd_tc_varlen over chunks of longer sequences (omlm_attn_fwd_tc_chunk): qn [M, heads*64] packed chunk rows, kv
    [rows, 128] (keys of sequence b at rows kv_start[b] ...); q_off int32 [n_seq] each chunk's first position; max_end >=
    every q_off + seq_len."""
    for t in (work, seq_start, seq_len, q_off, kv_start):
        assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous()
    assert kv.is_contiguous() and kv.shape[-1] == 128
    call("omlm_attn_fwd_tc_chunk", _p(qn), _p(kv), _L(kv.numel() // 128), _p(table), _I(table.stride(0)), _p(work), _I(work.numel() // 2),
         _p(seq_start), _p(seq_len), _p(q_off), _p(kv_start), _I(qn.shape[0]), _I(max_end), _p(out), _p(lse2), _I(heads), _F(scale),
         _stream())


def attn_bwd(qn, kvn, d_o, o, lse2, table, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads, scale=8.0):
    call("omlm_attn_bwd", _p(qn), _p(kvn), _p(d_o), _p(o), _p(lse2), _p(table), _I(table.stride(0)), _p(key_mask),
         _p(dsum_scratch), _p(dqn), _p(dkvn), _p(dtable), _I(B), _I(N), _I(heads), _F(scale), _stream())


def attn_bwd_tc(qn, kvn, d_o, o, lse2, table, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads, scale=8.0, det=None):
    """det: an AttnBwdDetWorkspace for this (B, N, heads) -> the fixed-order variant (omlm_attn_bwd_tc_det).
    dtable None: the variant without the bias gradient (dqn / dkvn as with a table)."""
    args = (_p(qn), _p(kvn), _p(d_o), _p(o), _p(lse2), _p(table), _I(table.stride(0)), _p(key_mask),
            _p(dsum_scratch), _p(dqn), _p(dkvn), _p(dtable), _I(B), _I(N), _I(heads), _F(scale))
    if det is None:
        call("omlm_attn_bwd_tc", *args, _stream())
    else:
        call("omlm_attn_bwd_tc_det", *args, _p(det.ws), _L(det.ws.numel() * 4), _p(det.iws), _L(det.iws.numel()), _stream())


class AttnBwdDetWorkspace:
    """Scratch of omlm_attn_bwd_tc_det for one (B, N, heads): the units' partial bias-gradient tables and the int words
    (turn counters, table windows, error word -- allocated zero)."""

    def __init__(self, device, B, N, heads):
        ws, iws = _L(0), _L(0)
        call("omlm_attn_bwd_tc_det_workspace", _I(B), _I(N), _I(heads), ctypes.byref(ws), ctypes.byref(iws))
        self.ws = torch.empty(max(ws.value // 4, 1), device=device, dtype=torch.float32)
        self.iws = torch.zeros(iws.value, device=device, dtype=torch.int32)

    def error(self):
        """True if a turn was not granted in time since the word was last cleared: those calls summed in arrival order
        (correct up to rounding, not reproducible).  Synchronises."""
        return bool(int(self.iws[-1].item()))

    def clear_error(self):
        self.iws[-1].zero_()


def gemm_ffn_up(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, Nseq, Fp, max_ctas=0):
    M, K = xn.shape
    assert xn.dtype in _T16 and xn.dtype == w1_packed.dtype == u_out.dtype == h_out.dtype
    call("omlm_gemm_ffn_up", _p(xn), _p(w1_packed), _p(conv_w_packed), _p(u_out), _p(h_out), _p(rowsum), _I(M), _I(Nseq),
         _I(K), _I(Fp), _I(int(xn.dtype == torch.float16)), _I(max_ctas), _stream())


def gemm_ffn_up_varlen(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, row_pos, Fp, max_ctas=0):
    """gemm_ffn_up over packed sequences (omlm_gemm_ffn_up_varlen): row_pos int32 [M], each row's position in its sequence."""
    M, K = xn.shape
    assert xn.dtype in _T16 and xn.dtype == w1_packed.dtype == u_out.dtype == h_out.dtype
    assert row_pos.dtype == torch.int32 and row_pos.is_cuda and row_pos.is_contiguous() and row_pos.numel() >= M
    call("omlm_gemm_ffn_up_varlen", _p(xn), _p(w1_packed), _p(conv_w_packed), _p(u_out), _p(h_out), _p(rowsum), _p(row_pos), _I(M),
         _I(K), _I(Fp), _I(int(xn.dtype == torch.float16)), _I(max_ctas), _stream())


def gemm_ffn_up_chunk(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, row_pos, hist, hist_idx, Fp, max_ctas=0):
    """gemm_ffn_up_varlen over chunks that continue longer sequences (omlm_gemm_ffn_up_chunk): hist [*, 2Fp] the history
    rows, hist_idx int32 [M] (c >= 0 at a chunk's first row: its t-2 and t-1 inputs are hist rows 2c and 2c + 1)."""
    M, K = xn.shape
    assert xn.dtype in _T16 and xn.dtype == w1_packed.dtype == u_out.dtype == h_out.dtype == hist.dtype
    assert hist.is_contiguous() and hist.shape[-1] == 2 * Fp
    for t in (row_pos, hist_idx):
        assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous() and t.numel() >= M
    call("omlm_gemm_ffn_up_chunk", _p(xn), _p(w1_packed), _p(conv_w_packed), _p(u_out), _p(h_out), _p(rowsum), _p(row_pos), _p(hist),
         _p(hist_idx), _I(M), _I(K), _I(Fp), _I(int(xn.dtype == torch.float16)), _I(max_ctas), _stream())


def ffn_norm_fwd(h, rowsum, gamma, hn, stats, F, Fp, drop_p=0.0, seed=None, layer=0, keep_bits=None, hn_copy=None):
    assert h.dtype in _T16 and h.dtype == hn.dtype and (hn_copy is None or hn_copy.dtype == torch.bfloat16)
    call("omlm_ffn_norm_fwd", _p(h), _p(rowsum), _p(gamma), _p(hn), _p(hn_copy), _p(stats), _p(keep_bits), _L(h.shape[0]),
         _I(F), _I(Fp), _F(drop_p), _p(seed), _I(layer), _I(int(h.dtype == torch.float16)), _stream())


def ffn_mid_bwd(dhn, hn, u, stats, conv_w, gamma, rowstat, du, dgamma, dconv_w, B, N, F, Fp, drop_p=0.0, keep_bits=None, rowstat_parts=0,
                part=None):
    """dgamma [F] / dconv_w [2F, 3] (each may be None: not summed) are accumulated in the parameters' own layouts;
    rowstat_parts > 0: rowstat holds the partial row sums written by gemm_rowstat, else it is a [M, 2] scratch."""
    assert u.dtype in _T16 and hn.dtype == dhn.dtype == du.dtype == torch.bfloat16
    assert (dgamma is None or dgamma.numel() == F) and (dconv_w is None or dconv_w.numel() == 6 * F)
    args = (_p(dhn), _p(hn), _p(u), _p(stats), _p(conv_w), _p(gamma), _p(keep_bits), _p(rowstat), _I(rowstat_parts), _p(du),
            _p(dgamma), _p(dconv_w), _I(B), _I(N), _I(F), _I(Fp), _F(drop_p), _I(int(u.dtype == torch.float16)))
    if part is None:
        call("omlm_ffn_mid_bwd", *args, _stream())
    else:
        call("omlm_ffn_mid_bwd_det", *args, _p(part), _L(part.numel() * 4), _stream())


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
                  rows_per_batch=0, batch_stride=0, loss_scale=1.0, part=None):
    """labels: int32; flat (rows_per_batch = 0) or the strided view described in include/omlm_b200.h (pass the tensor whose
    data_ptr is the first label of the group)."""
    rows = logits.shape[0] if rows is None else rows
    args = (_p(logits), _L(logits.stride(0)), _p(labels), _I(label_stride), _I(rows_per_batch), _L(batch_stride),
            _I(rows), _I(C), _I(ignore_index), _F(grad_scale), _F(loss_scale), _p(dlogits),
            _L(dlogits.stride(0) if dlogits is not None else 0), _I(dlogits.shape[1] if dlogits is not None else 0), _p(loss_acc))
    if part is None:
        call("omlm_cross_entropy", *args, _stream())
    else:
        call("omlm_cross_entropy_det", *args, _p(part), _L(part.numel() * 4), _stream())


def token_logprob(logits, labels, C, out, *, label_stride=1, rows=None, rows_per_batch=0, batch_stride=0):
    """out[r] (float32) = log softmax(logits[r, :C])[label_r] through omlm_token_logprob; labels int32 as in cross_entropy
    (a label outside [0, C) gives 0)."""
    rows = logits.shape[0] if rows is None else rows
    assert labels.dtype == torch.int32 and out.dtype == torch.float32 and out.numel() >= rows
    call("omlm_token_logprob", _p(logits), _L(logits.stride(0)), _p(labels), _I(label_stride), _I(rows_per_batch), _L(batch_stride),
         _I(rows), _I(C), _p(out), _stream())


def grad_sumsq(g, acc, prescale=1.0, part=None):
    """part: float64 scratch (>= 4 * SMs) -> the deterministic variant (omlm_grad_sumsq_det)."""
    if part is None:
        call("omlm_grad_sumsq", _p(g), _L(g.numel()), _F(prescale), _p(acc), _stream())
    else:
        call("omlm_grad_sumsq_det", _p(g), _L(g.numel()), _F(prescale), _p(acc), _p(part), _L(part.numel() * 8), _stream())


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


def decode_gemm_workspace(B, N, K, invariant=False):
    """Bytes of split-K partials omlm_decode_gemm (invariant: omlm_decode_gemm_invariant) needs for a B x N x K call on
    the current device."""
    part = _L(0)
    call("omlm_decode_gemm_invariant_workspace" if invariant else "omlm_decode_gemm_workspace", _I(B), _I(N), _I(K), ctypes.byref(part))
    return part.value


class DecodeWorkspace:
    """Scratch of the large-batch decode kernels, allocated once so that CUDA-graph capture allocates nothing:
    the 16-bit activation operand [B, max K], the split-K partials, the attention's per-slice partials and its
    per-sequence counters (zero; every call leaves them zero).  shapes: the (N, K) of every decode_gemm call; max_pos /
    heads: attention; invariant: also large enough for decode_gemm(..., invariant=True)."""

    def __init__(self, device, B, shapes, max_pos=0, heads=0, invariant=False):
        part = max(decode_gemm_workspace(B, N, K, inv) for N, K in shapes for inv in ((False, True) if invariant else (False,)))
        attn = B * -(-max_pos // 128) * heads * 66 if max_pos else 0
        self.a16 = torch.empty(B * max(K for _, K in shapes), device=device, dtype=torch.int16)
        self.part = torch.empty(max(part // 4, 1), device=device, dtype=torch.float32)
        self.attn = torch.empty(max(attn, 1), device=device, dtype=torch.float32)
        self.counters = torch.zeros(B, device=device, dtype=torch.int32)


def decode_gemm(A, W, out, *, prologue=0, gamma=None, rowsum=None, n_real=0, addend=None, ws=None, invariant=False):
    """skinny_gemm's contract for 1 <= B <= 256 rows on the tensor cores (omlm_decode_gemm).  ws: a DecodeWorkspace
    covering this shape (None: a fresh one, which is not CUDA-graph capturable).  invariant: the K split does not depend
    on B, so each output row is bit-identical for every batch size (omlm_decode_gemm_invariant)."""
    B = A.shape[0]
    N, K = W.shape
    assert W.dtype in _T16 and W.stride(1) == 1 and out.stride(-1) == 1 and A.stride(-1) == 1
    assert (prologue in (0, 3) and A.dtype == W.dtype) or (prologue in (1, 2) and A.dtype == torch.float32)
    if ws is None:
        ws = DecodeWorkspace(A.device, B, [(N, K)], invariant=invariant)
    call("omlm_decode_gemm_invariant" if invariant else "omlm_decode_gemm", _p(A), _L(A.stride(0)), _I(prologue), _p(W), _L(W.stride(0)), _I(int(W.dtype == torch.float16)),
         _p(gamma), _p(rowsum), _I(n_real), _p(addend), _L(addend.stride(0) if addend is not None else 0), _p(out),
         _I(FMT[out.dtype]), _L(out.stride(0)), _I(B), _I(N), _I(K), _p(ws.a16), _p(ws.part), _L(ws.part.numel() * 4),
         _stream())


def _check_row_pos(pos, B):
    assert pos.dtype == torch.int32 and pos.is_cuda and pos.is_contiguous() and pos.numel() >= B, "ragged: pos needs one int32 per row"


def attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, ws=None, scale=8.0, ragged=False):
    """attn_decode's contract with every cached row read once per sequence (omlm_attn_decode_mqa), 1 <= heads <= 16."""
    B = q_raw.shape[0]
    if ragged:
        _check_row_pos(pos, B)
    if ws is None:
        ws = DecodeWorkspace(q_raw.device, B, [(1, 8)], max_pos=max_pos, heads=heads)
    call("omlm_attn_decode_mqa_ragged" if ragged else "omlm_attn_decode_mqa", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale),
         _p(cache), _L(cache.stride(0)), _p(table),
         _I(table.stride(0)), _p(pos), _I(max_pos), _p(out), _I(B), _I(heads), _F(scale), _p(ws.attn), _L(ws.attn.numel() * 4),
         _p(ws.counters), _stream())


def attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, scale=8.0, ragged=False):
    """One decode step's attention at position pos[0] for every sequence (omlm_attn_decode); ragged: sequence b at its
    own position pos[b] (omlm_attn_decode_ragged, and likewise for attn_decode_mqa)."""
    if ragged:
        _check_row_pos(pos, q_raw.shape[0])
    call("omlm_attn_decode_ragged" if ragged else "omlm_attn_decode", _p(q_raw), _p(kv_raw), _p(q_scale), _p(k_scale), _p(cache),
         _L(cache.stride(0)), _p(table),
         _I(table.stride(0)), _p(pos), _I(max_pos), _p(out), _I(q_raw.shape[0]), _I(heads), _F(scale), _stream())


def decode_advance_pos(pos, pos_last):
    """pos[b] += 1 where pos[b] < pos_last[b] (int32 device tensors [B]; omlm_decode_advance_pos)."""
    assert pos.dtype == pos_last.dtype == torch.int32 and pos.is_contiguous() and pos_last.is_contiguous()
    assert pos.numel() == pos_last.numel()
    call("omlm_decode_advance_pos", _p(pos), _p(pos_last), _I(pos.numel()), _stream())


def decode_conv_geglu(u_new, state, conv_w, h_out, rowsum):
    B, Fp2 = u_new.shape
    assert u_new.dtype == state.dtype == h_out.dtype and u_new.dtype in _T16
    call("omlm_decode_conv_geglu", _p(u_new), _p(state), _p(conv_w), _p(h_out), _p(rowsum), _I(B), _I(Fp2 // 2),
         _I(int(u_new.dtype == torch.float16)), _stream())


def sample(logits, C, top_k, temperature, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B, seeds=None,
           top_p=None, top_k_rows=None, temperature_rows=None, top_p_rows=None, logprobs=None, sample_logprobs=None):
    """seeds: int64 [B] device tensor of per-sequence seeds (raw 64-bit patterns) -> omlm_sample_seeded.
    top_p: nucleus sampling (omlm_sample_nucleus, which rejects values outside (0, 1)); None or 1.0 samples over the
    whole top-k set through omlm_sample / omlm_sample_seeded.
    top_k_rows (int32 [B]), temperature_rows, top_p_rows (float32 [B]): per-sequence arguments (omlm_sample_rows); each
    one given replaces its scalar; top_p_rows selects the nucleus kernel and is the only way to pass top_p with them.
    logprobs, sample_logprobs (float32 [B, tokens' width]): also write each token's two log-probabilities
    (omlm_sample_logprob, the same tokens).  They must follow tokens in its allocation (tokens' B rows, then logprobs,
    then sample_logprobs; see logprob_buffers)."""
    if logprobs is not None:
        for t in (logprobs, sample_logprobs, top_k_rows, temperature_rows, top_p_rows):
            assert t is None or (t.dtype == (torch.int32 if t is top_k_rows else torch.float32) and t.is_cuda and t.is_contiguous())
        assert sample_logprobs is not None and logprobs.stride(0) == sample_logprobs.stride(0) == tokens.stride(0)
        assert seeds is None or (seeds.dtype == torch.int64 and seeds.is_contiguous() and seeds.numel() >= B)
        call("omlm_sample_logprob", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _p(top_k_rows), _F(temperature),
             _p(temperature_rows), _F(1.0 if top_p is None else top_p), _p(top_p_rows), _I(int(allow_eos)), _p(uniform), _p(seed),
             _p(seeds), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(counters), _p(pos), _I(B), _p(logprobs),
             _p(sample_logprobs), _stream())
        return
    if top_k_rows is not None or temperature_rows is not None or top_p_rows is not None:
        assert top_p is None or top_p == 1.0, "per-row sampling takes its nucleus masses through top_p_rows"
        for t, dt in ((top_k_rows, torch.int32), (temperature_rows, torch.float32), (top_p_rows, torch.float32)):
            assert t is None or (t.dtype == dt and t.is_cuda and t.is_contiguous() and t.numel() >= B)
        assert seeds is None or (seeds.dtype == torch.int64 and seeds.is_contiguous() and seeds.numel() >= B)
        call("omlm_sample_rows", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _p(top_k_rows), _F(temperature),
             _p(temperature_rows), _p(top_p_rows), _I(int(allow_eos)), _p(uniform), _p(seed), _p(seeds), _p(tokens),
             _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(counters), _p(pos), _I(B), _stream())
        return
    if top_p is not None and top_p != 1.0:
        assert seeds is None or (seeds.dtype == torch.int64 and seeds.is_contiguous() and seeds.numel() >= B)
        call("omlm_sample_nucleus", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _F(temperature), _F(top_p),
             _I(int(allow_eos)), _p(uniform), _p(seed), _p(seeds), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset),
             _p(counters), _p(pos), _I(B), _stream())
        return
    if seeds is None:
        call("omlm_sample", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _F(temperature), _I(int(allow_eos)), _p(uniform),
             _p(seed), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(counters), _p(pos), _I(B), _stream())
        return
    assert seeds.dtype == torch.int64 and seeds.is_contiguous() and seeds.numel() >= B
    call("omlm_sample_seeded", _p(logits), _L(logits.stride(0)), _I(C), _I(top_k), _F(temperature), _I(int(allow_eos)), _p(uniform),
         _p(seed), _p(seeds), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(counters), _p(pos), _I(B), _stream())


def logprob_buffers(B, W, device):
    """(tokens int64 [B, W], logprobs, sample_logprobs float32 [B, W]) in the one allocation the log-probability
    samplers require."""
    store = torch.zeros(2 * B * W, device=device, dtype=torch.int64)
    lp, slp = store[B * W:].view(torch.float32).view(2, B, W).unbind(0)
    return store[:B * W].view(B, W), lp, slp


def sample_rows_indexed(logits, C, allow_eos, seeds, tokens, next_row, row_offset, step_rows, n_rows, top_k_rows, temperature_rows,
                        top_p_rows=None, logprobs=None, sample_logprobs=None):
    """omlm_sample_rows_indexed: sequence b samples its token at its own index t = step_rows[b] (int32 [B]) under
    seeds[b] (int64 [B]) while t < n_rows[b] (int32 [B]) and then sets step_rows[b] = t + 1; per-row top_k_rows (int32),
    temperature_rows and top_p_rows (float32, None: no row narrows to a nucleus) as in omlm_sample_rows.
    logprobs, sample_logprobs: as in sample (omlm_sample_rows_indexed_logprob)."""
    B = logits.shape[0]
    for t, dt in ((seeds, torch.int64), (step_rows, torch.int32), (n_rows, torch.int32), (top_k_rows, torch.int32),
                  (temperature_rows, torch.float32), (top_p_rows, torch.float32)):
        assert t is None or (t.dtype == dt and t.is_cuda and t.is_contiguous() and t.numel() >= B)
    if logprobs is not None:
        assert sample_logprobs is not None and logprobs.stride(0) == sample_logprobs.stride(0) == tokens.stride(0)
        assert logprobs.dtype == sample_logprobs.dtype == torch.float32
        call("omlm_sample_rows_indexed_logprob", _p(logits), _L(logits.stride(0)), _I(C), _I(1), _p(top_k_rows), _F(1.0),
             _p(temperature_rows), _p(top_p_rows), _I(int(allow_eos)), _p(seeds), _p(tokens), _L(tokens.stride(0)), _p(next_row),
             _I(row_offset), _p(step_rows), _p(n_rows), _I(B), _p(logprobs), _p(sample_logprobs), _stream())
        return
    call("omlm_sample_rows_indexed", _p(logits), _L(logits.stride(0)), _I(C), _I(1), _p(top_k_rows), _F(1.0), _p(temperature_rows),
         _p(top_p_rows), _I(int(allow_eos)), _p(seeds), _p(tokens), _L(tokens.stride(0)), _p(next_row), _I(row_offset), _p(step_rows),
         _p(n_rows), _I(B), _stream())


def gather_windows(src_i16, start, out):
    """out[b, t, c] = src[(start[b] + t), c] for a flat [T_total, width] int16 token store (ids are uint16)."""
    B, length = out.shape[0], out.shape[1]
    width = src_i16.shape[1] if src_i16.dim() == 2 else 1
    assert src_i16.dtype == torch.int16 and start.dtype == torch.int64 and out.dtype == torch.int64 and out.is_contiguous()
    call("omlm_gather_windows", _p(src_i16), _p(start), _p(out), _I(length), _I(width), _I(B), _stream())
