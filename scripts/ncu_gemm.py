"""One GEMM shape, a few launches — the target of `ncu --set full` (run under gpurun)."""
import math, sys, torch
sys.path.insert(0, ".")
from kubeai_b200 import ops
T, N, K = (int(a) for a in sys.argv[1:4])
x = torch.randn(T, K, device="cuda").bfloat16()
w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
mode = sys.argv[4] if len(sys.argv) > 4 else "plain"
if mode == "gemm3_silu":      # the decode path's dominant launch: gate_up with the SiLU*up epilogue
    fn = lambda x, w: ops.gemm3(x, w, epi=ops.EPI_SILU)
elif mode == "gemm3_resadd":  # o_proj / down_proj: cluster split-K, residual add + fused RMSNorm
    res = torch.randn(T, N, device="cuda").bfloat16()
    nw = torch.ones(N, device="cuda").bfloat16()
    fn = lambda x, w: ops.gemm3(x, w, epi=ops.EPI_RESADD, out=res, norm_w_out=nw)
elif mode == "gemm3":
    fn = lambda x, w: ops.gemm3(x, w)
else:
    fn = ops.gemm_deferred if mode == "deferred" else ops.gemm
for _ in range(4):
    flush.zero_()
    fn(x, w)
torch.cuda.synchronize()
