"""Debug helper: stage timestamps of tc_forward_kernel (UAVRL_TC_TRACE=1 python tools/tc_trace.py)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import uavrl_b200
from uavrl_b200 import engine
L = engine.Learner(100, [64, 64], 27, False, 0, batch_size=4096, replay_capacity=8192)
L.init_params(0)
x = torch.randn(4096, 100, device="cuda")
for _ in range(5):
    L.act(x, 0.1)
torch.cuda.synchronize()
# training kernels: [tc_trace] lines for the TD pass and [dw_trace] for the weight-gradient kernel (a layer-0 and a layer-1 CTA)
B = 4096
s = torch.randn(B, 100, device="cuda"); s2 = torch.randn(B, 100, device="cuda")
a = torch.randint(0, 27, (B,), device="cuda", dtype=torch.int32); r = torch.randn(B, device="cuda"); d = torch.zeros(B, device="cuda")
for _ in range(3):
    L.update_batch(s, a, r, s2, d)
torch.cuda.synchronize()
