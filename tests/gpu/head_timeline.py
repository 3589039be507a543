"""Per-CTA event timeline (SM cycles) of the fused classifier-head kernel, hot and in a graph-like loop."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_yarn_b200.keras import fastpath  # noqa: E402,F401
from tf_yarn_b200.ops import native  # noqa: E402

lib = native.load()
native.declare("tfy_nn_set_timeline", [ctypes.c_void_p])
dev = "cuda"
B, K, C = 128, 128, 10
h = torch.randn(B, K, device=dev).relu().bfloat16()
w2 = (torch.randn(C, K, device=dev) * 0.2).bfloat16()
b2 = torch.zeros(C, device=dev).bfloat16()
y = torch.randint(0, C, (B,), device=dev)
mask = (torch.rand(B, K, device=dev) > 0.4).to(torch.uint8)
loss = torch.zeros((), device=dev)
stats = torch.zeros(2, device=dev)
dw2 = torch.zeros(C, K, dtype=torch.bfloat16, device=dev)
db2 = torch.zeros(C, dtype=torch.bfloat16, device=dev)
dh = torch.zeros(B, K, dtype=torch.bfloat16, device=dev)
db1 = torch.zeros(K, dtype=torch.bfloat16, device=dev)
scratch = torch.zeros(int(lib.tfy_dense_head_scratch_elems(K, C, B)), device=dev)
counter = torch.zeros(1, dtype=torch.int32, device=dev)


def run():
    return lib.tfy_dense_head_fused(h.data_ptr(), w2.data_ptr(), b2.data_ptr(), y.data_ptr(), mask.data_ptr(),
                                    ctypes.c_float(2.0), loss.data_ptr(), None, stats.data_ptr(), dw2.data_ptr(),
                                    db2.data_ptr(), dh.data_ptr(), db1.data_ptr(), scratch.data_ptr(),
                                    counter.data_ptr(), B, K, C, torch.cuda.current_stream().cuda_stream)


for _ in range(5):
    run()
torch.cuda.synchronize()
tl = torch.zeros(16 * 16, dtype=torch.int64, device=dev)
lib.tfy_nn_set_timeline(tl.data_ptr())
run()
torch.cuda.synchronize()
lib.tfy_nn_set_timeline(None)
v = tl.view(16, 16)[:8].cpu()
names = ["-", "staged", "softmax_done", "dW2_reds_issued", "dh_done", "fence_done", "counter_done", "end"]
for j in range(1, 8):
    print(f"{names[j]:>18}: median {int(v[:, j].float().median())} max {int(v[:, j].max())}")
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    for _ in range(20):
        run()
g.replay()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    g.replay()
e1.record()
torch.cuda.synchronize()
print("head fused us/launch (graph)", e0.elapsed_time(e1) * 10.0)
