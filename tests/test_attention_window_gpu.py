"""The wgmma attention kernels read the relative-position bias from a per-tile Toeplitz window in shared memory and
fold the causal mask into it.  These cases pin that window's geometry against the mma.sync reference kernels at the
tolerances of test_kernels_gpu.py: the full cfg2 shape (many tiles per unit), a short tailed sequence with fewer CTAs
than SMs, one head (the widest window) and 12 heads (row tiles that start mid-position), with a bias table wider than N."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("B,N,h", [(16, 1024, 8), (1, 200, 8), (2, 300, 1), (1, 260, 12)])
def test_window_matches_mma_sync_reference(B, N, h):
    from open_musiclm_b200 import lib
    torch.manual_seed(7 * N + h)
    M = B * N
    qn = F.normalize(torch.randn(M, h, 64, device=DEV), dim=-1).reshape(M, h * 64).bfloat16()
    kv = torch.randn(M, 128, device=DEV)
    kv[:, :64] = F.normalize(kv[:, :64], dim=-1)
    kvn = kv.bfloat16()
    table = (0.05 * torch.randn(h, 1, device=DEV) * torch.arange(N + 40, device=DEV)[None]
             + 0.3 * torch.randn(h, N + 40, device=DEV)).contiguous()
    key_mask = (torch.rand(B, N, device=DEV) > 0.2).to(torch.uint8)
    key_mask[:, 0] = 1
    out = torch.empty(M, h * 64, device=DEV, dtype=torch.bfloat16)
    lse = torch.empty(B, N * h, device=DEV)
    lib.attn_fwd(qn, kvn, table, key_mask, out, lse, B, N, h)
    out_tc = torch.full_like(out, float("nan"))
    lse_tc = torch.full_like(lse, float("nan"))
    lib.attn_fwd_tc(qn, kvn, table, key_mask, out_tc, lse_tc, B, N, h)
    torch.cuda.synchronize()
    assert rel(out_tc, out) < 6e-3, rel(out_tc, out)
    assert float((lse_tc - lse).abs().max()) < 2e-2

    d_o = torch.randn(M, h * 64, device=DEV).bfloat16()
    dsum = torch.empty(M * h, device=DEV)
    dq = torch.zeros(M, h * 64, device=DEV); dkv = torch.zeros(M, 128, device=DEV); dt = torch.zeros_like(table)
    lib.attn_bwd(qn, kvn, d_o, out, lse, table, key_mask, dsum, dq, dkv, dt, B, N, h)
    ws = lib.AttnBwdDetWorkspace(DEV, B, N, h)
    for det in (None, ws):
        dq2 = torch.full_like(dq, float("nan")); dkv2 = torch.full_like(dkv, float("nan")); dt2 = torch.zeros_like(table)
        lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, dsum, dq2, dkv2, dt2, B, N, h, det=det)
        torch.cuda.synchronize()
        assert rel(dq2, dq) < 1.5e-2, (det is not None, rel(dq2, dq))
        assert rel(dkv2, dkv) < 1.5e-2, (det is not None, rel(dkv2, dkv))
        assert rel(dt2[:, :N], dt[:, :N]) < 1.5e-2, (det is not None, rel(dt2[:, :N], dt[:, :N]))
        assert float(dt2[:, N:].abs().max()) == 0.0
    assert not ws.error()


def test_rows_without_a_visible_key_get_zero_gradients():
    """With the leading keys masked, the first positions see no key at all (lse2 = -inf).  Their P must be 0, not
    exp2(-inf - -inf) = NaN: the backward keeps the causal compare even though the window holds the bias."""
    from open_musiclm_b200 import lib
    B, N, h = 2, 200, 8
    torch.manual_seed(3)
    M = B * N
    qn = F.normalize(torch.randn(M, h, 64, device=DEV), dim=-1).reshape(M, h * 64).bfloat16()
    kv = torch.randn(M, 128, device=DEV)
    kv[:, :64] = F.normalize(kv[:, :64], dim=-1)
    kvn = kv.bfloat16()
    table = 0.3 * torch.randn(h, N, device=DEV)
    key_mask = torch.ones(B, N, device=DEV, dtype=torch.uint8)
    key_mask[:, :3] = 0
    out = torch.empty(M, h * 64, device=DEV, dtype=torch.bfloat16)
    lse = torch.empty(B, N * h, device=DEV)
    lib.attn_fwd_tc(qn, kvn, table, key_mask, out, lse, B, N, h)
    assert torch.isinf(lse.view(B, N, h)[:, :3]).all() and torch.isfinite(lse.view(B, N, h)[:, 3:]).all()
    d_o = torch.randn(M, h * 64, device=DEV).bfloat16()
    dsum = torch.empty(M * h, device=DEV)
    ws = lib.AttnBwdDetWorkspace(DEV, B, N, h)
    for det in (None, ws):
        dq = torch.empty(M, h * 64, device=DEV); dkv = torch.empty(M, 128, device=DEV); dt = torch.zeros_like(table)
        lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, dsum, dq, dkv, dt, B, N, h, det=det)
        torch.cuda.synchronize()
        assert torch.isfinite(dq).all() and torch.isfinite(dkv).all() and torch.isfinite(dt).all(), det is not None
        assert float(dq.view(B, N, -1)[:, :3].abs().max()) == 0.0
        assert float(dkv.view(B, N, -1)[:, :3].abs().max()) == 0.0      # masked keys get no gradient
    assert not ws.error()


def test_too_many_heads_for_the_windows_is_an_error():
    from open_musiclm_b200 import lib
    B, N, h = 1, 64, 128
    qn = torch.zeros(B * N, h * 64, device=DEV, dtype=torch.bfloat16)
    kvn = torch.zeros(B * N, 128, device=DEV, dtype=torch.bfloat16)
    table = torch.zeros(h, N, device=DEV)
    out = torch.empty_like(qn)
    lse = torch.empty(B, N * h, device=DEV)
    with pytest.raises(lib.OmlmError, match="too many heads"):
        lib.attn_fwd_tc(qn, kvn, table, None, out, lse, B, N, h)
