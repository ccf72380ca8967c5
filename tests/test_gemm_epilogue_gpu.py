"""The GEMM's staged epilogue (tile results through shared memory, TMA stores, addend and hn by TMA loads) against a
float64 reference, and against the direct-store epilogue of the same build, which a launch takes when an output row
pitch is not 16-byte aligned.  Row tails (M not a multiple of 128), column tails (n_valid < N, N not a multiple of the
tile width) and the in-place weight gradient (addend == out) are covered.  A column tail that does not end on a 16-byte
boundary (n_valid = 90, 513) also takes the direct epilogue: TMA clips stores only at 16-byte granularity."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 3.0


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm().clamp_min(1e-12)).item()


def _padded(rows, cols, pad, dtype=torch.float32, fill=SENTINEL):
    """A [rows, cols + pad] buffer filled with `fill`, for a GEMM of `cols` columns (pad 8: 16-byte-aligned rows; pad 1: not)."""
    return torch.full((rows, cols + pad), fill, device="cuda", dtype=dtype)


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K,n_valid", [(1000, 1032, 520, 1000), (4100, 1024, 512, 1024), (128, 96, 64, 88), (300, 520, 1000, 456),
                                           (128, 96, 64, 90), (300, 520, 1000, 513)])
def test_staged_epilogue_matches_float64_and_direct(block_n, M, N, K, n_valid):
    from open_musiclm_b200 import lib
    torch.manual_seed(M + N + K + block_n)
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = torch.randn(N, K, device="cuda").bfloat16()
    X = torch.randn(M, N, device="cuda")
    prod = A.double() @ B.double().t()
    for dtype, tol in ((torch.bfloat16, 6e-3), (torch.float32, 1e-5)):
        outs = []
        for pad in (8, 1):
            buf = _padded(M, N, pad, dtype)
            lib.gemm(A, B, buf, N=N, n_valid=n_valid, block_n=block_n)
            outs.append(buf)
        torch.cuda.synchronize()
        staged, direct = outs
        assert _rel(staged[:, :n_valid], prod[:, :n_valid]) < tol
        assert torch.equal(staged[:, :n_valid], direct[:, :n_valid])
        assert bool((staged[:, n_valid:] == SENTINEL).all())       # columns past n_valid and the pitch padding stay untouched
    # fp32 output with the residual addend and alpha != 1
    outs = []
    for pad in (8, 1):
        xb = _padded(M, N, pad)
        xb[:, :N] = X
        buf = _padded(M, N, pad)
        lib.gemm(A, B, buf, N=N, n_valid=n_valid, addend=xb, alpha=0.5, block_n=block_n)
        outs.append(buf)
    torch.cuda.synchronize()
    ref = (0.5 * prod + X.double())[:, :n_valid]
    assert _rel(outs[0][:, :n_valid], ref) < 1e-5
    assert torch.equal(outs[0][:, :n_valid], outs[1][:, :n_valid])
    assert bool((outs[0][:, n_valid:] == SENTINEL).all())


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(1000, 1032, 520), (300, 520, 1000), (1024, 2816, 4096)])
def test_staged_epilogue_inplace_weight_gradient(block_n, M, N, K):
    """gout[M, N] += dy^T x with both operands MN-major and the gradient as its own addend (one tile per CTA reads the
    rows it then overwrites), staged against direct and float64."""
    from open_musiclm_b200 import lib
    torch.manual_seed(M * 3 + N + K + block_n)
    mp = (M + 7) // 8 * 8                       # 16-byte-aligned operand rows
    dy = torch.randn(K, mp, device="cuda").bfloat16()[:, :M]
    x = torch.randn(K, N, device="cuda").bfloat16()
    G = torch.randn(M, N, device="cuda")
    ref = G.double() + dy.double().t() @ x.double()
    outs = []
    for pad in (8, 1):
        g = _padded(M, N, pad)
        g[:, :N] = G
        lib.gemm(dy, x, g, a_mn=True, b_mn=True, M=M, N=N, K=K, addend=g, block_n=block_n)
        outs.append(g)
    torch.cuda.synchronize()
    assert _rel(outs[0][:, :N], ref) < 1e-5
    assert torch.equal(outs[0][:, :N], outs[1][:, :N])
    assert bool((outs[0][:, N:] == SENTINEL).all())


@pytest.mark.parametrize("M,N,K,p", [(1000, 512, 520, 0.0), (4100, 768, 256, 0.25), (2048, 2816, 1024, 0.1)])
def test_staged_rowstat_against_float64(M, N, K, p):
    """d_hn = a b (bf16, through the staged epilogue with hn loaded by TMA) and its per-128-column partial row sums
    (sum gamma * drop(d), sum d * hn) against float64 sums of the same fp32 d values."""
    from open_musiclm_b200 import lib
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(K, N, device="cuda").bfloat16()
    hn = torch.randn(M, N, device="cuda").bfloat16()
    gamma = torch.randn(N, device="cuda")
    keep = torch.randint(0, 256, (M, N // 8), device="cuda", dtype=torch.uint8) if p > 0 else None
    scale = 1.0 / (1.0 - p)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    part = torch.full((M * (N // 128) * 2,), float("nan"), device="cuda")
    lib.gemm_rowstat(a, b, out, hn, gamma, part, b_mn=True, M=M, N=N, K=K, keep_bits=keep, keep_scale=scale)
    torch.cuda.synchronize()
    d = a.double() @ b.double()
    assert _rel(out, d) < 6e-3
    if keep is None:
        mask = torch.ones(M, N, device="cuda", dtype=torch.float64)
    else:
        bits = (keep.long().unsqueeze(-1) >> torch.arange(8, device="cuda")) & 1
        mask = bits.reshape(M, N).double()
    s1 = (gamma.double() * mask * d).reshape(M, N // 128, 128).sum(-1) * scale
    s2 = (d * hn.double()).reshape(M, N // 128, 128).sum(-1)
    got = part.reshape(M, N // 128, 2).double()
    # fp32 accumulation of 128 products of fp32 d values: bounded by the sum of magnitudes
    b1 = (gamma.double().abs() * mask * d.abs()).reshape(M, N // 128, 128).sum(-1) * scale * 1e-5 + 1e-6
    b2 = (d.abs() * hn.double().abs()).reshape(M, N // 128, 128).sum(-1) * 1e-5 + 1e-6
    assert bool(((got[..., 0] - s1).abs() <= b1).all()), float(((got[..., 0] - s1).abs() / b1).max())
    assert bool(((got[..., 1] - s2).abs() <= b2).all()), float(((got[..., 1] - s2).abs() / b2).max())
