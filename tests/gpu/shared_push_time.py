"""Time the deep tower's sparse push with shared embedding columns against unshared tables (CUDA events).

    python tests/gpu/shared_push_time.py [out_dir]

Shapes of bench/wide_deep.py (batch 512, 26 hashed columns of 100k buckets, 13 numerics, deep embeddings of 64, hidden
1024-512-256), with the 26 deep columns either as 13 shared pairs (c0 with c13, c1 with c14, ...: 13 tables) or as 26
embedding columns (26 tables).  It reports:
  push      : the deep tower's push alone, as K5's backward runs it on the first layer's bf16 dx
              (tfy_ps_multi_push_rows_shared on 13 tables against tfy_ps_multi_push_rows on 26): CUDA events over
              back-to-back calls, and each of its kernels' device time from torch.profiler;
  step      : one single-GPU worker step (pull, forward, backward, push) through the HBM plane over a local buffer
              standing in for the ps rank's shard, shared against unshared, alternated;
  launches  : kernel launches per step of both, as the connection counts them;
  card      : name, power limit and max SM clock, read in the same run.
"""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from feature_ids_time import _card, _time  # noqa: E402
from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.estimator import canned, ps, ps_hbm  # noqa: E402
from tf_yarn_b200.estimator import feature_column as fc  # noqa: E402
from tf_yarn_b200.models import wide_deep as wdm  # noqa: E402

B, V, N_CAT, N_NUM, HIDDEN = 512, 100_000, 26, 13, [1024, 512, 256]


def _deep(shared):
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=N_CAT, n_num=N_NUM)
    if not shared:
        return wide, deep
    cats = [c.categorical_column for c in deep if isinstance(c, fc.EmbeddingColumn)]
    half = N_CAT // 2
    pairs = [fc.shared_embedding_columns([cats[i], cats[i + half]], 64) for i in range(half)]
    emb = [p[0] for p in pairs] + [p[1] for p in pairs]          # column order c0..c25, as the unshared tower
    return wide, emb + [c for c in deep if not isinstance(c, fc.EmbeddingColumn)]


def _plane(net, tmp, tag):
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05)
    layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05),
                            {n: ftrl for n, _ in named if n.startswith("linear.")})
    region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
    import types
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


def _deep_push(net, conn, feats):
    """K5's push of the deep tables, alone: the group K5 builds (one pointer per column), its one-hot ids and a random
    bf16 dx of the first layer's width, pushed back to back."""
    df, lin = net.dense_features, net.hidden[0]
    by_param = {id(p): i for i, p in enumerate(conn.params)}
    emb = [c for c in df.columns if isinstance(c, (fc.EmbeddingColumn, fc.SharedEmbeddingColumn))]
    idx = [by_param[id(df.embeddings[fc._embedding_key(c)].weight)] for c in emb]
    group = ps_hbm._TableGroup(conn, idx, [c.categorical_column for c in emb], 64, 64)
    ids = group.ids_of(feats)
    Kp = conn.shadow_ld(by_param[id(lin.weight)])
    dx = (torch.randn(B, Kp, device="cuda") * 1e-3).to(torch.bfloat16)

    def push():
        group.push(ids, dx, dout_ld=Kp)
    out = {"entry_point": "tfy_ps_multi_push_rows_shared" if group.shared else "tfy_ps_multi_push_rows",
           "tables": len(group.distinct), "max_members": group.max_members if group.shared else 1,
           "events_us_per_push": _time(push, 2000)}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(100):
            push()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name] = per.get(e.name, 0.0) + e.device_time_total / 100
    out["kernel_device_us_per_push"] = per
    out["device_us_per_push"] = sum(per.values())
    return out


def main(out_dir):
    torch.manual_seed(0)
    feats, y = wdm.synthetic_batches(B, 1, vocab=V, seed=1, n_cat=N_CAT, n_num=N_NUM)[0]
    feats = {k: v.cuda() for k, v in feats.items()}
    y = y.cuda().float()
    planes = {}
    with tempfile.TemporaryDirectory() as tmp:
        for shared in (True, False):
            wide, deep = _deep(shared)
            net = canned._WideDeepNet(wide, deep, HIDDEN, 1).cuda()
            planes[shared] = (net,) + _plane(net, tmp, "shared" if shared else "unshared")

        def step(shared):
            net, conn = planes[shared][0], planes[shared][1]
            conn.pull(net)
            net.zero_grad(set_to_none=False)
            out = net(feats).float()
            torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y).backward()
            conn.push(net)

        step_us = {True: [], False: []}
        for _ in range(3):                                  # alternated, to see the spread
            for shared in (True, False):
                step_us[shared].append(_time(lambda: step(shared), 100))
        launches, push_us = {}, {}
        for shared in (True, False):
            step(shared)
            torch.cuda.synchronize()
            launches[shared] = planes[shared][1].traffic_per_step()["launches_per_step"]
            push_us[shared] = _deep_push(planes[shared][0], planes[shared][1], feats)
        for shared in (True, False):
            planes[shared][2].unlink()
    out = {"card": _card(), "shapes": {"B": B, "deep_columns": N_CAT, "V": V, "D": 64, "numerics": N_NUM,
                                       "shared_tables": N_CAT // 2, "unshared_tables": N_CAT},
           "push": {"shared_pairs": push_us[True], "unshared": push_us[False]},
           "step_us": {"shared_pairs": step_us[True], "unshared": step_us[False]},
           "launches_per_step_counted": {"shared_pairs": launches[True], "unshared": launches[False]}}
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "shared_push_time.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
