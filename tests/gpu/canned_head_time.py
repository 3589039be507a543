"""What the canned head kernel (tfy_canned_head) costs and saves against the torch statement of the same loss.

    python tests/gpu/canned_head_time.py [out_dir]

It reports, with the card's name, power limit and max SM clock read in the same run:
  head      : the head's forward + backward alone (loss, then .backward() into a leaf), kernel against the torch
              statement (ops/head.py torch_head on CUDA tensors), binary / multi-class (C = 10) / regression (d = 1),
              weighted and not, at B = 512, 4096, 65536: CUDA-event time per call over many calls, and the summed
              device time of its kernels from torch.profiler in a separate run;
  kernels   : CUDA kernels (graph nodes) of one wide-and-deep worker step of bench/wide_deep.py's shapes (batch 512,
              26 hashed columns of 100k buckets, 13 numerics, embeddings of 64, hidden 1024-512-256; K5 and the fused
              wide tower) with each head, counted with torch.profiler in a run of their own;
  step      : that worker step (pull, forward, head, backward, push through the HBM plane over a local buffer standing
              in for the ps rank's shard), captured in a CUDA graph as the estimator does and replayed; every
              configuration timed three times, alternated, so the spread shows.
"""
import json
import os
import subprocess
import sys
import tempfile
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.estimator import canned, ps, ps_hbm  # noqa: E402
from tf_yarn_b200.models import wide_deep as wdm  # noqa: E402
from tf_yarn_b200.ops import head as H  # noqa: E402

B_STEP, V, N_CAT, N_NUM, HIDDEN = 512, 100_000, 26, 13, [1024, 512, 256]
HEADS = {"binary": (H.BINARY, 1), "multiclass": (H.MULTI_CLASS, 10), "regression": (H.REGRESSION, 1)}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def _time(fn, reps):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def _kernels(fn, n=5):
    """(kernels per call, summed kernel device time per call in us) from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(ev) / n, sum(e.device_time_total for e in ev) / n


def _loss_fn(impl, head, n_out):
    if impl == "kernel":
        return H.CannedHead(head, n_out)
    return lambda y, z, w=None: H.torch_head(head, z, y, w)


def _inputs(head, n_out, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, n_out, generator=g) * 3
    if head == H.BINARY:
        y = (torch.rand(B, generator=g) < 0.3).long()
    elif head == H.MULTI_CLASS:
        y = torch.randint(0, n_out, (B,), generator=g)
    else:
        y = torch.randn(B, generator=g)
    w = torch.rand(B, generator=g) * 2
    return z.cuda(), y.cuda(), w.cuda()


def head_alone():
    out = []
    for name, (head, n_out) in HEADS.items():
        for B in (512, 4096, 65536):
            z0, y, w = _inputs(head, n_out, B)
            z = z0.clone().requires_grad_(True)
            for weighted in (False, True):
                row = {"head": name, "B": B, "weighted": weighted}
                for impl in ("torch", "kernel"):
                    loss = _loss_fn(impl, head, n_out)

                    def call():
                        z.grad = None
                        (loss(y, z, w) if weighted else loss(y, z)).backward()
                    row[f"{impl}_us"] = round(_time(call, 300), 2)
                    k, dev = _kernels(call)
                    row[f"{impl}_kernels"] = k
                    row[f"{impl}_device_us"] = round(dev, 2)
                out.append(row)
    return out


def _plane(net, tmp, tag):
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05)
    layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05),
                            {n: ftrl for n, _ in named if n.startswith("linear.")})
    region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
    comm = types.SimpleNamespace(arena=types.SimpleNamespace(peer_base={0: region.data_ptr()}), device=0)
    header = ps.ShmShard(os.path.join(tmp, f"header_{tag}"), 8, create=True)
    conn = ps_hbm.HbmConnection(layout, comm, {"ps:0": 0}, 0, [n for n, _ in named], header, net)
    with torch.no_grad():
        for i, (_, p) in enumerate(named):
            conn.remote_tensor(i).copy_(p.detach().reshape(-1))
            if layout.kinds[i] in ("adagrad", "ftrl"):
                conn.remote_tensor(i, 1).fill_(layout.hypers[i]["init_s1"])
    conn.refresh_shadows()
    header.set_global_step(0)
    conn.install(net)
    assert conn.fused_first and conn.fused_wide
    return conn, header, region


def worker_step():
    torch.manual_seed(0)
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=N_CAT, n_num=N_NUM)
    feats, yb = wdm.synthetic_batches(B_STEP, 1, vocab=V, seed=1, n_cat=N_CAT, n_num=N_NUM)[0]
    feats = {k: v.cuda() for k, v in feats.items()}
    feats["weight"] = (torch.rand(B_STEP) * 2).cuda()
    yb, c0 = yb.cuda(), feats["c0"][:, 0]                 # [B] labels, [B] ids of the first hashed column
    labels = {"binary": yb, "multiclass": (yb * 3 + c0 % 3) % 10, "regression": feats["numeric"][:, 0] * 2 + yb.float()}
    for y in labels.values():
        assert y.shape == (B_STEP,), y.shape
    configs = [(name, impl, weighted) for name in HEADS for impl in ("torch", "kernel") for weighted in (False, True)]
    res = {"kernels_per_step": {}, "step_us": {}, "errors": {}}
    with tempfile.TemporaryDirectory() as tmp:
        planes = {}
        for n_out in sorted({n for _, n in HEADS.values()}):
            net = canned._WideDeepNet(wide, deep, HIDDEN, n_out).cuda()
            planes[n_out] = (net,) + _plane(net, tmp, n_out)
        steps = {}
        for name, impl, weighted in configs:
            head, n_out = HEADS[name]
            net, conn = planes[n_out][0], planes[n_out][1]
            loss_fn = _loss_fn(impl, head, n_out)
            y = labels[name]

            def body(net=net, conn=conn, loss_fn=loss_fn, y=y, weighted=weighted):
                conn.pull(net)
                net.zero_grad(set_to_none=False)
                out = net(feats)
                loss = loss_fn(y, out, feats["weight"]) if weighted else loss_fn(y, out)
                loss.backward()
                conn.push(net)
                return loss.detach()
            key = f"{name}/{impl}/{'weighted' if weighted else 'unweighted'}"
            k, _ = _kernels(body, 3)
            res["kernels_per_step"][key] = k
            for _ in range(3):
                body()
            torch.cuda.synchronize()
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    body()
                steps[key] = g.replay
            except Exception as exc:  # noqa: BLE001  (reported, the step stays eager)
                res["errors"][key] = f"{type(exc).__name__}: {exc}"[:300]
                steps[key] = body
        for key in steps:
            res["step_us"][key] = []
        for _ in range(3):                                  # alternated, to see the spread
            for key, fn in steps.items():
                res["step_us"][key].append(round(_time(fn, 200), 1))
        for n_out in planes:
            planes[n_out][2].unlink()
    return res


def main(out_dir):
    if not torch.cuda.is_available():
        raise SystemExit("canned_head_time.py needs a GPU")
    torch.cuda.set_device(0)
    out = {"card": _card(), "head": head_alone()}
    print(json.dumps(out, indent=1), flush=True)
    out.update(worker_step=worker_step(),
               step_shapes={"B": B_STEP, "hashed": N_CAT, "V": V, "numerics": N_NUM, "hidden": HIDDEN})
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "canned_head_time.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
