"""wgmma GEMM (csrc/gemm_tc.cu) vs a plain torch fp32 reference of the same contraction."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (384, 640, 512), (1000, 1032, 520), (128, 128, 64)])
def test_gemm_majors(a_mn, b_mn, block_n, M, N, K):
    from open_musiclm_b200 import lib
    torch.manual_seed(M * 7 + N * 3 + K)
    dev = "cuda"
    A = torch.randn(M, K, device=dev).bfloat16()
    B = torch.randn(N, K, device=dev).bfloat16()
    ref = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    for dtype in (torch.bfloat16, torch.float32):
        out = torch.full((M, N), float("nan"), device=dev, dtype=dtype)
        lib.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, block_n=block_n)
        torch.cuda.synchronize()
        err = _rel(out, ref)
        assert err < (6e-3 if dtype == torch.bfloat16 else 1e-5), (a_mn, b_mn, block_n, M, N, K, dtype, err)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_gemm_fp16_operands(a_mn, b_mn):
    """wgmma with fp16 operands (the .f16 instruction form) — the forward GEMMs of the hot path.
    Mixed fp16 x bf16 is rejected on the host: one wgmma takes a single operand format."""
    from open_musiclm_b200 import lib
    torch.manual_seed(11)
    M, N, K = 384, 640, 520
    # values that tell the formats apart: fp16 keeps 11 significant bits, bf16 8
    A = (torch.randn(M, K, device="cuda") * 1.37).half()
    B = (torch.randn(N, K, device="cuda") * 0.71).half()
    ref = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    for bn in (128, 256):
        out = torch.full((M, N), float("nan"), device="cuda")
        lib.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, block_n=bn)
        torch.cuda.synchronize()
        err = _rel(out, ref)
        assert err < 1e-5, (a_mn, b_mn, bn, err)      # exact products of the stored fp16 values, fp32 accumulate
    with pytest.raises(lib.OmlmError):
        lib.gemm(a.bfloat16(), b, out, a_mn=a_mn, b_mn=b_mn)


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(1000, 1032, 520), (128, 96, 64), (4100, 1024, 512)])
def test_gemm_residual_tma_epilogue_tails(block_n, M, N, K):
    """fp32 output + fp32 addend through the shared-memory staged epilogue (TMA loads of the addend, TMA stores) with row and
    column tails, out of place and in place (128-wide tiles prefetch the addend two chunks ahead, 256-wide ones reuse one buffer)."""
    from open_musiclm_b200 import lib
    torch.manual_seed(M + N + K + block_n)
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = torch.randn(N, K, device="cuda").bfloat16()
    X = torch.randn(M, N, device="cuda")
    ref = X + A.float() @ B.float().t()
    guard = torch.full((M + 2, N), 7.0, device="cuda")          # rows beyond M must stay untouched
    out = guard[:M]
    lib.gemm(A, B, out, addend=X, block_n=block_n)
    assert _rel(out, ref) < 1e-5 and float((guard[M:] - 7.0).abs().max()) == 0.0
    x2 = X.clone()
    lib.gemm(A, B, x2, addend=x2, block_n=block_n)
    assert _rel(x2, ref) < 1e-5


def test_gemm_residual_and_splitk():
    from open_musiclm_b200 import lib
    torch.manual_seed(1)
    M, N, K = 512, 1024, 2816
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = torch.randn(N, K, device="cuda").bfloat16()
    X = torch.randn(M, N, device="cuda")
    ref = X + A.float() @ B.float().t()
    out = torch.empty_like(X)
    lib.gemm(A, B, out, addend=X)
    assert _rel(out, ref) < 1e-5
    x2 = X.clone()
    lib.gemm(A, B, x2, addend=x2)  # in place
    assert _rel(x2, ref) < 1e-5
    # split-K atomics accumulate on top of existing contents
    acc = X.clone()
    lib.gemm(A, B, acc, splits=5)
    assert _rel(acc, ref) < 1e-5
    # weight-gradient form: dW[N,K'] = dY[M,N]^T X[M,K'] with both operands MN-major, into a padded layout
    dY = torch.randn(M, 256, device="cuda").bfloat16()
    Xa = torch.randn(M, 384, device="cuda").bfloat16()
    dW = torch.zeros(200, 300, device="cuda")  # canonical (unpadded) gradient: 2 halves of 100 rows, 300 cols
    lib.gemm(dY, Xa, dW, a_mn=True, b_mn=True, splits=3, row_split=128, row_valid=100, n_valid=300)
    full = dY.float().t() @ Xa.float()
    ref_dw = torch.cat([full[0:100, :300], full[128:228, :300]], 0)
    assert _rel(dW, ref_dw) < 1e-5
    # interleaved GEGLU row order (groups of 128 channels: value rows | gate rows), F = 200 of Fp = 256
    dY2 = torch.randn(M, 512, device="cuda").bfloat16()
    dW2 = torch.zeros(400, 300, device="cuda")
    lib.gemm(dY2, Xa, dW2, a_mn=True, b_mn=True, splits=2, row_split=-1, row_valid=200, n_valid=300)
    full2 = dY2.float().t() @ Xa.float()            # packed rows: [0:128 value ch 0-127 | 128:256 gate ch 0-127 | 256:384 value ch 128-255 | ...]
    val = torch.cat([full2[0:128], full2[256:256 + 72]], 0)[:, :300]
    gate = torch.cat([full2[128:256], full2[384:384 + 72]], 0)[:, :300]
    assert _rel(dW2, torch.cat([val, gate], 0)) < 1e-5


def test_gemm_large_timing():
    """Not a benchmark: just makes sure the FFN-up shape of cfg2 runs and is correct on a sample."""
    from open_musiclm_b200 import lib
    torch.manual_seed(2)
    M, N, K = 16384, 5632, 1024
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = torch.randn(N, K, device="cuda").bfloat16()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    for bn in (128, 256):
        lib.gemm(A, B, out, block_n=bn)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            lib.gemm(A, B, out, block_n=bn)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        print(f"gemm {M}x{N}x{K} bn={bn}: {ms:.3f} ms  {2 * M * N * K / ms / 1e9:.1f} TFLOP/s")
        idx = torch.randint(0, M, (64,), device="cuda")
        ref = A[idx].float() @ B.float().t()
        assert _rel(out[idx], ref) < 6e-3
