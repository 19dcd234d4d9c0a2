"""Driver for an ncu source-level capture of the CTA-pair GEMM on an epilogue-bound shape
(M = N = 8192, K = 64: 13.8 tiles per cluster, one k-block each) and on a single-wave shape with a residual epilogue.

  ncu --set full --import-source on --clock-control none -k regex:gemm_wgmma -s 4 -c 2 -o epi \
      python tools/ncu_epi.py"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch

from magma_b200 import ops

dev = torch.device("cuda:0")
A = torch.randn(8192, 64, device=dev).to(torch.bfloat16)
B = (torch.randn(8192, 64, device=dev) * 0.05).to(torch.bfloat16)
C = torch.empty(8192, 8192, device=dev, dtype=torch.bfloat16)
A2 = torch.randn(1024, 4096, device=dev).to(torch.bfloat16)
B2 = (torch.randn(4096, 4096, device=dev) * 0.05).to(torch.bfloat16)
R = torch.randn(1024, 4096, device=dev).to(torch.bfloat16)
C2 = torch.empty(1024, 4096, device=dev, dtype=torch.bfloat16)
for _ in range(3):
    ops.gemm(A, B, out=C, force_bn=512)          # launches 0, 2, 4
    ops.gemm(A2, B2, out=C2, res1=R, b_static=True)  # launches 1, 3, 5
torch.cuda.synchronize()
print("done")
