"""What the multi-label, Poisson and logistic heads of tfy_canned_head cost against the torch statement of the same loss.

    python tests/gpu/head_kinds_time.py [out_dir]

It reports, with the card's name, power limit and max SM clock read in the same run:
  head      : the head's forward + backward alone (loss, then .backward() into a leaf), kernel against the torch
              statement (ops/head.py torch_head on CUDA tensors), multi-label at C = 2, 10, 100, 1000, Poisson (d = 1,
              with and without the full loss) and logistic, weighted and not, at B = 512, 4096, 65536: CUDA-event time
              per call over many calls, and kernels per call with their summed device time from torch.profiler in a
              separate run;
  step      : the wide-and-deep worker step of canned_head_time.py (bench/wide_deep.py's shapes, B = 512, K5 and the
              fused wide tower, captured in a CUDA graph and replayed) under MultiLabelHead(4), kernel against the torch
              statement, weighted and not, with kernels per step; every configuration timed three times, alternated.
"""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

import canned_head_time as cht  # noqa: E402
from tf_yarn_b200.estimator import canned  # noqa: E402
from tf_yarn_b200.models import wide_deep as wdm  # noqa: E402
from tf_yarn_b200.ops import head as H  # noqa: E402

HEADS = [("multi_label", H.MULTI_LABEL, C) for C in (2, 10, 100, 1000)] + \
    [("poisson", H.POISSON, 1), ("poisson_full", H.POISSON_FULL, 1), ("logistic", H.LOGISTIC, 1)]
STEP_C = 4


def _inputs(head, n_out, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, n_out, generator=g) * 2
    if head == H.MULTI_LABEL:
        y = (torch.rand(B, n_out, generator=g) < 0.3).long()
    elif head == H.LOGISTIC:
        y = torch.rand(B, generator=g)
    else:
        y = torch.poisson(torch.full((B,), 3.0), generator=g)
    w = torch.rand(B, generator=g) * 2
    return z.cuda(), y.cuda(), w.cuda()


def head_alone():
    out = []
    for name, head, n_out in HEADS:
        for B in (512, 4096, 65536):
            z0, y, w = _inputs(head, n_out, B)
            z = z0.clone().requires_grad_(True)
            for weighted in (False, True):
                row = {"head": name, "C": n_out, "B": B, "weighted": weighted}
                for impl in ("torch", "kernel"):
                    loss = cht._loss_fn(impl, head, n_out)

                    def call():
                        z.grad = None
                        (loss(y, z, w) if weighted else loss(y, z)).backward()
                    row[f"{impl}_us"] = round(cht._time(call, 300), 2)
                    k, dev = cht._kernels(call)
                    row[f"{impl}_kernels"] = k
                    row[f"{impl}_device_us"] = round(dev, 2)
                out.append(row)
    return out


def worker_step():
    torch.manual_seed(0)
    wide, deep = wdm.feature_columns(vocab=cht.V, emb_dim=64, n_cat=cht.N_CAT, n_num=cht.N_NUM)
    feats, yb = wdm.synthetic_batches(cht.B_STEP, 1, vocab=cht.V, seed=1, n_cat=cht.N_CAT, n_num=cht.N_NUM)[0]
    feats = {k: v.cuda() for k, v in feats.items()}
    feats["weight"] = (torch.rand(cht.B_STEP) * 2).cuda()
    yb = yb.cuda().reshape(-1, 1)
    cols = torch.stack([feats[f"c{j}"][:, 0] % 2 for j in range(STEP_C - 1)], dim=1)
    y = torch.cat([yb, cols], dim=1)                         # [B, 4]: the click and three id-derived tags
    res = {"kernels_per_step": {}, "step_us": {}, "errors": {}}
    with tempfile.TemporaryDirectory() as tmp:
        net = canned._WideDeepNet(wide, deep, cht.HIDDEN, STEP_C).cuda()
        conn, header, region = cht._plane(net, tmp, "ml")   # region: the shard conn points into, kept alive
        steps = {}
        for impl in ("torch", "kernel"):
            for weighted in (False, True):
                loss_fn = cht._loss_fn(impl, H.MULTI_LABEL, STEP_C)

                def body(loss_fn=loss_fn, weighted=weighted):
                    conn.pull(net)
                    net.zero_grad(set_to_none=False)
                    out = net(feats)
                    loss = loss_fn(y, out, feats["weight"]) if weighted else loss_fn(y, out)
                    loss.backward()
                    conn.push(net)
                    return loss.detach()
                key = f"multi_label/{impl}/{'weighted' if weighted else 'unweighted'}"
                k, _ = cht._kernels(body, 3)
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
        for _ in range(3):                                   # alternated, to see the spread
            for key, fn in steps.items():
                res["step_us"][key].append(round(cht._time(fn, 200), 1))
        header.unlink()
        del region
    return res


def main(out_dir):
    if not torch.cuda.is_available():
        raise SystemExit("head_kinds_time.py needs a GPU")
    torch.cuda.set_device(0)
    out = {"card": cht._card(), "head": head_alone()}
    print(json.dumps(out, indent=1), flush=True)
    out.update(worker_step=worker_step(),
               step_shapes={"B": cht.B_STEP, "hashed": cht.N_CAT, "V": cht.V, "numerics": cht.N_NUM,
                            "hidden": cht.HIDDEN, "C": STEP_C})
    print(json.dumps(out["worker_step"], indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "head_kinds_time.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
