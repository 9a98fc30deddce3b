"""Profiling driver: the three pixel-parallel ops of one optimisation step at the BASELINE
shape, called through the C ABI a few times (for a profiler run of its own)."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from flowmap_b200 import ops  # noqa: E402
from flowmap_b200._lib import lib  # noqa: E402

F, H, W = (int(x) for x in (sys.argv[1:4] if len(sys.argv) >= 4 else (150, 360, 640)))
REPS = int(sys.argv[4]) if len(sys.argv) >= 5 else 3
KMODE = int(sys.argv[5]) if len(sys.argv) >= 6 else 1  # FM_K_SHARED_FOCAL, as the fused step uses
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
depths = (0.1 + 0.05 * torch.rand(1, F, H, W, device=dev, generator=g))
weights = torch.sigmoid(torch.randn(1, F - 1, H, W, device=dev, generator=g))
fwd = 0.01 * torch.randn(1, F - 1, H, W, 2, device=dev, generator=g)
bwd = 0.01 * torch.randn(1, F - 1, H, W, 2, device=dev, generator=g)
fm = torch.rand(1, F - 1, H, W, device=dev, generator=g)
bm = torch.rand(1, F - 1, H, W, device=dev, generator=g)
s = (H * W) ** 0.5
k4 = torch.tensor([0.85 * s / W, 0.85 * s / H, 0.5, 0.5], device=dev).expand(1, F, 4).contiguous()
msum = ops.mask_sum(fm, bm)
ws = ops.workspace(1, F, H, W, dev)
rt = torch.empty(1, F - 1, 3, 4, device=dev)
g_depth, g_w, g_k4, g_rt = (torch.empty_like(depths), torch.empty_like(weights),
                            torch.empty_like(k4), torch.empty_like(rt))
loss = torch.empty((), device=dev)
P = lambda x: x.data_ptr()  # noqa: E731
st = torch.cuda.current_stream().cuda_stream
L = lib()
for _ in range(REPS):
    L.fm_procrustes_fwd(P(depths), P(k4), P(bwd), P(weights), None, 0, P(rt), P(ws), 1, F, H, W, st)
    L.fm_flow_loss_fwd_bwd(P(depths), P(k4), P(rt), P(fwd), P(bwd), P(fm), P(bm), P(msum), 0, 0.01,
                           1000.0, KMODE, P(loss), P(g_depth), P(g_rt), P(g_k4), P(ws), 1, F, H, W, st)
    L.fm_procrustes_bwd(P(depths), P(k4), P(bwd), P(weights), None, 0, None, 1, None, P(g_depth),
                        P(g_w), P(g_k4), P(ws), 1, F, H, W, st)
torch.cuda.synchronize()
print("loss", float(loss))
