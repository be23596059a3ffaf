"""Bring-up probe for the tensor-core GEMM (run by hand on a GPU, not a pytest test): structured inputs whose
output reveals operand-layout / descriptor mistakes."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import capi   # noqa: E402

lib = capi.load()
tag = sys.argv[1] if len(sys.argv) > 1 else "default"


def run(a, w, name):
    M, K = a.shape
    N = w.shape[0]
    d = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    rc = lib.ds_test_gemm_bf16(capi.DS_GEMM_TCGEN05, a.data_ptr(), w.data_ptr(), None, d.data_ptr(), M, N, K, 0, None)
    if rc:
        print(name, "FAILED", lib.ds_last_error().decode())
        return None
    ref = a.float() @ w.float().t()
    err = (d.float() - ref).abs().max().item()
    print("%s [%s]: M=%d N=%d K=%d max_err=%.4g ref_max=%.4g" % (name, tag, M, N, K, err, ref.abs().max().item()))
    return err


# 1. A = identity on the first 64 k: D[m, n] = W[n, m] for m < 64
a = torch.zeros(128, 64, dtype=torch.bfloat16)
a[:64, :64] = torch.eye(64)
w = (torch.arange(128 * 64).reshape(128, 64).float() % 251 / 16).to(torch.bfloat16)
run(a.cuda(), w.cuda(), "a_identity")
# 2. W = identity: D[m, n] = A[m, n] for n < 64
a2 = (torch.arange(128 * 64).reshape(128, 64).float() % 241 / 16).to(torch.bfloat16)
w2 = torch.zeros(128, 64, dtype=torch.bfloat16)
w2[:64, :64] = torch.eye(64)
run(a2.cuda(), w2.cuda(), "w_identity")
# 3. random, one k-block / many k-blocks / N=256 tile / multi-tile
g = torch.Generator().manual_seed(0)
for (M, N, K) in [(128, 128, 64), (128, 128, 256), (128, 256, 64), (128, 256, 512), (512, 512, 512),
                  (1000, 384, 512), (20000, 512, 1024)]:
    a = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(torch.bfloat16)
    run(a.cuda(), w.cuda(), "rand_%d_%d_%d" % (M, N, K))
print("probe done")
