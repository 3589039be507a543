"""Time the bucket-id preparation of a wide tower with bucketized and crossed columns (CUDA events).

    python tests/gpu/feature_ids_time.py [out_dir]

Shapes of bench/wide_deep.py (batch 512, 26 hashed columns of 100k buckets, 13 numerics, deep embeddings of 64, hidden
1024-512-256), with the wide tower extended by the 13 numerics bucketized at 10 boundaries each and 8 pairwise crosses
of the hashed columns into 10k buckets (T = 35 tables, so two tfy_feature_ids launches).  It reports:
  ids          : the tower's [T, B, L] ids by tfy_feature_ids against the torch statement of the columns on the same
                 device tensors, over many calls; the kernel's bytes (sources read, ids written) against the HBM floor
                 at 3.35 TB/s;
  step         : one single-GPU worker step (pull, forward, backward, push) through the HBM plane over a local buffer
                 standing in for the ps rank's shard, wide tower fused against TFY_PS_FUSE_WIDE=0, alternated;
  launches     : kernel launches per step of both, as the connection counts them;
  card         : name, power limit and max SM clock, read in the same run.
"""
import copy
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
from tf_yarn_b200.estimator import feature_column as fc  # noqa: E402
from tf_yarn_b200.models import wide_deep as wdm  # noqa: E402
from tf_yarn_b200.ops import features as feature_ids  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

B, V, N_CAT, N_NUM, HIDDEN = 512, 100_000, 26, 13, [1024, 512, 256]
HBM_BYTES_PER_S = 3.35e12


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


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def _columns():
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=N_CAT, n_num=N_NUM)
    nb = fc.bucketized_column(fc.numeric_column("numeric", (N_NUM,)), [-2.0 + 0.4 * i for i in range(10)])
    crosses = [fc.crossed_column([f"c{2 * i}", f"c{2 * i + 1}"], 10_000) for i in range(8)]
    return wide + [nb] + crosses, deep


def _plane(net, layout, named, tmp, fuse_wide):
    region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
    comm = types.SimpleNamespace(arena=types.SimpleNamespace(peer_base={0: region.data_ptr()}), device=0)
    header = ps.ShmShard(os.path.join(tmp, f"header{int(fuse_wide)}"), 8, create=True)
    conn = ps_hbm.HbmConnection(layout, comm, {"ps:0": 0}, 0, [n for n, _ in named], header, net)
    with torch.no_grad():
        for i, (_, p) in enumerate(named):
            conn.remote_tensor(i).copy_(p.detach().reshape(-1))
            if layout.kinds[i] in ("adagrad", "ftrl"):
                conn.remote_tensor(i, 1).fill_(layout.hypers[i]["init_s1"])
    conn.refresh_shadows()
    header.set_global_step(0)
    os.environ["TFY_PS_FUSE_WIDE"] = "1" if fuse_wide else "0"
    conn.install(net)
    os.environ.pop("TFY_PS_FUSE_WIDE")
    assert conn.fused_wide == fuse_wide and conn.fused_first
    return conn, header, region


def main(out_dir):
    lib = native.load()
    torch.manual_seed(0)
    wide, deep = _columns()
    feats, y = wdm.synthetic_batches(B, 1, vocab=V, seed=1, n_cat=N_CAT, n_num=N_NUM)[0]
    feats = {k: v.cuda() for k, v in feats.items()}
    y = y.cuda().float()

    # ---- id preparation alone
    cat_cols = [fc._categorical(c) for c in wide if fc._categorical(c) is not None]
    builder = feature_ids.FeatureIds(cat_cols, torch.device("cuda"))
    kernel_ids = builder(feats, lib)
    torch_ids = torch.stack([torch.nn.functional.pad(i, (0, kernel_ids.shape[2] - i.shape[1]), value=-1)
                             for i in (fc._ids_and_weights(c, feats)[0] for c in cat_cols)])
    torch.cuda.synchronize()
    assert torch.equal(kernel_ids, torch_ids)
    T, _, L = kernel_ids.shape
    src_bytes = sum(v.numel() * v.element_size() for k, v in feats.items())
    out_bytes = T * B * L * 8
    ids = {"T": T, "L_max": L, "launches": builder.launches,
           "kernel_us": _time(lambda: builder(feats, lib), 2000),
           "torch_us": _time(lambda: [fc._ids_and_weights(c, feats) for c in cat_cols], 200),
           "bytes": src_bytes + out_bytes, "hbm_floor_us": (src_bytes + out_bytes) / HBM_BYTES_PER_S * 1e6}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            builder(feats, lib)
        torch.cuda.synchronize()
    dev_us = [e.device_time_total for e in prof.events()
              if e.device_type == torch.autograd.DeviceType.CUDA and "tfy_feature_ids" in e.name]
    ids["kernel_device_us_per_call"] = sum(dev_us) / 20

    # ---- whole worker step, fused wide tower against TFY_PS_FUSE_WIDE=0
    net_ref = canned._WideDeepNet(wide, deep, HIDDEN, 1)
    planes = {}
    with tempfile.TemporaryDirectory() as tmp:
        for fuse in (True, False):
            net = copy.deepcopy(net_ref).cuda()
            named = ps._named_trainables(net)
            ftrl = keras.optimizers.Ftrl(0.05)
            layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05),
                                    {n: ftrl for n, _ in named if n.startswith("linear.")})
            planes[fuse] = (net,) + _plane(net, layout, named, tmp, fuse)

        def step(fuse):
            net, conn = planes[fuse][0], planes[fuse][1]
            conn.pull(net)
            net.zero_grad(set_to_none=False)
            out = net(feats).float()
            torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y).backward()
            conn.push(net)

        step_us = {True: [], False: []}
        for _ in range(3):                                  # alternated, to see the spread
            for fuse in (True, False):
                step_us[fuse].append(_time(lambda: step(fuse), 100))
        launches = {}
        for fuse in (True, False):
            step(fuse)
            torch.cuda.synchronize()
            launches[fuse] = planes[fuse][1].traffic_per_step()["launches_per_step"]
        for fuse in (True, False):
            planes[fuse][2].unlink()
    out = {"card": _card(), "shapes": {"B": B, "hashed": N_CAT, "V": V, "numerics": N_NUM, "bucketized_boundaries": 10,
                                       "crosses": 8, "cross_V": 10_000},
           "ids": ids,
           "step_us": {"fused_wide": step_us[True], "unfused_wide": step_us[False]},
           "launches_per_step_counted": {"fused_wide": launches[True], "unfused_wide": launches[False]}}
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "feature_ids_time.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
