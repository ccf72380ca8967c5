"""Device time of the attention kernels at the BASELINE shapes (CUDA events, 20 launches after warm-up)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch, torch.nn.functional as F
from open_musiclm_b200 import lib


def run(B, N, h, tag):
    M = B * N
    torch.manual_seed(0)
    qn = F.normalize(torch.randn(M, h, 64, device="cuda"), dim=-1).reshape(M, h * 64).bfloat16()
    kvn = torch.randn(M, 128, device="cuda").bfloat16()
    table = (torch.randn(h, 1, device="cuda") * 0.05 * torch.arange(N, device="cuda")[None]).contiguous()
    km = (torch.rand(B, N, device="cuda") > 0.15).to(torch.uint8); km[:, 0] = 1
    out = torch.empty(M, h * 64, device="cuda", dtype=torch.bfloat16); lse = torch.empty(B, N * h, device="cuda")
    d_o = torch.randn(M, h * 64, device="cuda").bfloat16()
    dqn = torch.zeros(M, h * 64, device="cuda"); dkvn = torch.zeros(M, 128, device="cuda"); dtab = torch.zeros_like(table)
    dsum = torch.empty(M * h, device="cuda")
    fl = 2.0 * 2 * 64 * B * N * h * (N + 1) / 2          # causal forward flops (QK^T + PV)

    def t(fn, n=20):
        for _ in range(3): fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n): fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n * 1e3
    us_f = t(lambda: lib.attn_fwd_tc(qn, kvn, table, km, out, lse, B, N, h))
    us_b = t(lambda: lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, km, dsum, dqn, dkvn, dtab, B, N, h))
    det = lib.AttnBwdDetWorkspace("cuda", B, N, h)
    us_d = t(lambda: lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, km, dsum, dqn, dkvn, dtab, B, N, h, det=det))
    assert not det.error()
    print(f"{tag}: B={B} N={N} h={h}  fwd {us_f:.1f} us ({fl / us_f / 1e6:.0f} TF/s)   bwd {us_b:.1f} us ({2.5 * fl / us_b / 1e6:.0f} TF/s)"
          f"   bwd det {us_d:.1f} us ({2.5 * fl / us_d / 1e6:.0f} TF/s)", flush=True)


if __name__ == "__main__":
    run(16, 1024, 8, "cfg2")
    run(8, 2048, 8, "cfg3")
    run(16, 1024, 16, "cfg4")
