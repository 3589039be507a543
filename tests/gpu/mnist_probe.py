"""Probe: how fast is the MNIST-CNN step with stock PyTorch pieces on H100?

Design input for the mini-Keras train step (which ops are worth replacing).
Times eager vs CUDA-graphed fwd+bwd(+optimizer) in bf16 at batch 128.
"""
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.c1 = nn.Conv2d(1, 32, 3)
        self.c2 = nn.Conv2d(32, 64, 3)
        self.f1 = nn.Linear(9216, 128)
        self.f2 = nn.Linear(128, 10)

    def forward(self, x):
        x = F.relu(self.c1(x))
        x = F.relu(self.c2(x))
        x = F.max_pool2d(x, 2)
        x = F.dropout(x, 0.25, self.training)
        x = torch.flatten(x, 1)
        x = F.relu(self.f1(x))
        x = F.dropout(x, 0.5, self.training)
        return self.f2(x)


def timeit(fn, iters=200, warm=20):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3  # us


def main():
    torch.backends.cudnn.benchmark = True
    dev = "cuda"
    out = {}
    for B in (128, 1024):
        for mode in ("autocast_bf16", "pure_bf16", "pure_bf16_cl"):
            torch.manual_seed(0)
            net = Net().to(dev)
            x = torch.randn(B, 1, 28, 28, device=dev)
            y = torch.randint(0, 10, (B,), device=dev)
            if mode.startswith("pure"):
                net = net.to(torch.bfloat16)
                x = x.to(torch.bfloat16)
            if mode.endswith("_cl"):
                net = net.to(memory_format=torch.channels_last)
                x = x.contiguous(memory_format=torch.channels_last)
            opt = torch.optim.Adadelta(net.parameters(), lr=1.0, capturable=True) if False else \
                torch.optim.Adadelta(net.parameters(), lr=1.0)

            def fwdbwd():
                if mode == "autocast_bf16":
                    with torch.autocast("cuda", dtype=torch.bfloat16):
                        loss = F.cross_entropy(net(x).float(), y)
                else:
                    loss = F.cross_entropy(net(x).float(), y)
                loss.backward()
                return loss

            def step():
                opt.zero_grad(set_to_none=False)
                fwdbwd()
                opt.step()

            us_eager = timeit(step, 100, 10)
            # graphed fwd+bwd only (optimizer replaced by our fused kernel in the real engine)
            for p in net.parameters():
                p.grad = torch.zeros_like(p)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(3):
                    fwdbwd()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fwdbwd()
            us_graph = timeit(g.replay, 200, 20)
            out[f"B{B}/{mode}"] = {"eager_step_us": us_eager, "graph_fwdbwd_us": us_graph}
            print(f"B={B} {mode}: eager step {us_eager:.1f} us, graphed fwd+bwd {us_graph:.1f} us", flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open("gpurun_out/mnist_probe.json", "w"), indent=1)


if __name__ == "__main__":
    sys.exit(main())
