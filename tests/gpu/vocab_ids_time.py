"""Time the vocabulary lookup of a wide tower of vocabulary columns (CUDA events and torch.profiler).

    python tests/gpu/vocab_ids_time.py [out_dir]

26 vocabulary columns at batch 512, each with its own vocabulary of V random 32-bit keys and 3 OOV buckets; each
column's raw values are Zipf-skewed (exponent 1.1) over its keys, with about 10 % replaced by values outside the
vocabulary.  It reports:
  ids       : per V in (1e5, 1e6), the device time per call of the group's tfy_vocab_ids and tfy_feature_ids launches
              (torch.profiler, its own pass), the time per call of the whole FeatureIds call (CUDA events, host
              included), the host time of filling its launch descriptors alone (FeatureIds.prepare, perf_counter),
              and the torch statement of the columns on the same device tensors (CUDA events), three runs each;
  step      : one single-GPU worker step (pull, forward, backward, push) through the HBM plane over a local buffer
              standing in for the ps rank's shard, V = 1e5, wide tower fused against TFY_PS_FUSE_WIDE=0, alternated;
  launches  : kernel launches per step of both, as the connection counts them;
  card      : name, power limit and max SM clock, read in the same run.
"""
import copy
import json
import os
import subprocess
import sys
import tempfile
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.estimator import canned, ps, ps_hbm  # noqa: E402
from tf_yarn_b200.estimator import feature_column as fc  # noqa: E402
from tf_yarn_b200.ops import features as feature_ids  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

B, N_COLS, N_NUM, HIDDEN, OOV_BUCKETS, OOV_SHARE = 512, 26, 13, [1024, 512, 256], 3, 0.10


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


def _host_time(fn, reps):
    """Host time per call of host-only work (filling the launch descriptors), in microseconds."""
    for _ in range(10):
        fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) * 1e6 / reps


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def _columns_and_batch(V, seed=0):
    g = np.random.default_rng(seed)
    cols, feats = [], {}
    for i in range(N_COLS):
        keys = g.choice(2 ** 32, V + V // 10, replace=False).astype(np.int64)
        vocab, outside = keys[:V], keys[V:]
        cols.append(fc.categorical_column_with_vocabulary_list(f"c{i}", vocab, num_oov_buckets=OOV_BUCKETS))
        rank = np.minimum(g.zipf(1.1, B), V) - 1
        raw = vocab[rank]
        miss = g.random(B) < OOV_SHARE
        raw[miss] = outside[g.integers(0, outside.size, int(miss.sum()))]
        feats[f"c{i}"] = torch.from_numpy(raw.reshape(B, 1))
    feats["numeric"] = torch.from_numpy(g.standard_normal((B, N_NUM)).astype(np.float32))
    return cols, feats


def _profile(fn, names, calls=20):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for name in names:
        us = [e.device_time_total for e in prof.events()
              if e.device_type == torch.autograd.DeviceType.CUDA and name in e.name]
        out[name] = sum(us) / calls
    return out


def _ids(lib, V):
    cols, feats = _columns_and_batch(V)
    feats = {k: v.cuda() for k, v in feats.items()}
    fi = feature_ids.FeatureIds(cols, "cuda")
    kernel = fi(feats, lib)
    torch_ids = torch.stack([fc._ids_and_weights(c, feats)[0] for c in cols])
    torch.cuda.synchronize()
    assert torch.equal(kernel, torch_ids)
    oov = float(((kernel >= V) | (kernel < 0)).float().mean())
    out = {"V": V, "launches": fi.launches, "oov_share": round(oov, 4),
           "call_us": [_time(lambda: fi(feats, lib), 2000) for _ in range(3)],
           "prepare_host_us": [_host_time(lambda: fi.prepare(feats), 2000) for _ in range(3)],
           "torch_us": [_time(lambda: [fc._ids_and_weights(c, feats) for c in cols], 200) for _ in range(3)]}
    out["device_us_per_call"] = _profile(lambda: fi(feats, lib), ["tfy_vocab_ids", "tfy_feature_ids"])
    return out


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


def _steps(V):
    torch.manual_seed(0)
    cols, feats = _columns_and_batch(V, seed=1)
    feats = {k: v.cuda() for k, v in feats.items()}
    y = (feats["numeric"][:, 0] > 0).float()
    wide = [fc.numeric_column("numeric", (N_NUM,))] + cols
    deep = [fc.embedding_column(c, 64) for c in cols] + [fc.numeric_column("numeric", (N_NUM,))]
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
    return ({"V": V, "fused_wide": step_us[True], "unfused_wide": step_us[False]},
            {"fused_wide": launches[True], "unfused_wide": launches[False]})


def main(out_dir):
    lib = native.load()
    card = _card()
    ids = [_ids(lib, V) for V in (100_000, 1_000_000)]
    step_us, launches = _steps(100_000)
    out = {"card": card, "shapes": {"B": B, "vocabulary_columns": N_COLS, "oov_buckets": OOV_BUCKETS,
                                    "oov_share": OOV_SHARE, "zipf": 1.1, "numerics": N_NUM, "hidden": HIDDEN},
           "ids": ids, "step_us": step_us, "launches_per_step_counted": launches}
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "vocab_ids_time.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
