import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch, torch.nn.functional as F
from open_musiclm_b200 import lib
h = 8
for (B, N) in [(16, 1024), (4, 2048), (1, 4096), (64, 512), (16, 2048), (2, 1024), (132, 128), (132, 256), (132, 1024)]:
    M = B * N
    qn = F.normalize(torch.randn(M, h, 64, device="cuda"), dim=-1).reshape(M, h * 64).bfloat16()
    kvn = torch.randn(M, 128, device="cuda").bfloat16()
    table = (torch.randn(h, 1, device="cuda") * 0.05 * torch.arange(N, device="cuda")[None]).contiguous()
    km = torch.ones(B, N, device="cuda", dtype=torch.uint8)
    out = torch.empty(M, h * 64, device="cuda", dtype=torch.bfloat16); lse = torch.empty(B, N * h, device="cuda")
    for name, fn in (("mma", lib.attn_fwd), ("tc", lib.attn_fwd_tc)):
        for _ in range(3): fn(qn, kvn, table, km, out, lse, B, N, h)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10): fn(qn, kvn, table, km, out, lse, B, N, h)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        ctas = ((N * h + 255) // 256) * B
        print(f"B={B:4d} N={N:5d} {name:4s} {ms*1000:8.1f} us  ctas={ctas:5d}  {B * N * h * 64 * (N + 1) * 2 / ms / 1e9:6.0f} TFLOP/s")
