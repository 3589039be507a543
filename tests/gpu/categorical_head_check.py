"""Multi-GPU check of the fast path's dense-target classifier head.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29641 \
        tests/gpu/categorical_head_check.py

Every rank fits the MNIST CNN (hvd.DistributedOptimizer(Adadelta), 50 steps of its own 128-sample batches) twice:
with CategoricalCrossentropy(from_logits=True) on one-hot targets and with SparseCategoricalCrossentropy(from_logits=
True) on the labels, without and with sample / class weights.  The two runs must give the same per-step losses,
epoch logs and parameter bits, and the parameters must be the same on every rank.
"""
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

STEPS = 50


def fit(loss, x, y, **kw):
    from tf_yarn_b200 import hvd, keras
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
    torch.manual_seed(7)
    m = keras_mnist_cnn()
    m.compile(loss=loss, optimizer=hvd.DistributedOptimizer(keras.optimizers.Adadelta(1.0)), metrics=["accuracy"],
              weighted_metrics=["accuracy"] if kw else None)
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    hist = m.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0, callbacks=[Rec()], **kw)
    torch.cuda.synchronize()
    return m, losses, hist.history


def params_in_sync(t):
    ref = t.clone()
    dist.broadcast(ref, 0)
    flag = torch.tensor([1 if torch.equal(ref, t) else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from tf_yarn_b200 import hvd, keras
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    from tf_yarn_b200.models.mnist_cnn import synthetic_mnist
    hvd.init()
    x, y = synthetic_mnist(128 * STEPS, seed=100 + rank)
    onehot = torch.nn.functional.one_hot(y, 10).float()
    ok = True
    for name, kw in (("plain", {}),
                     ("weighted", {"sample_weight": torch.rand(len(y), generator=torch.Generator().manual_seed(rank)),
                                   "class_weight": {c: 0.25 + 0.3 * c for c in range(10)}})):
        sparse = fit(keras.losses.SparseCategoricalCrossentropy(from_logits=True), x, y, **kw)
        cat = fit(keras.losses.CategoricalCrossentropy(from_logits=True), x, onehot, **kw)
        fast = all(isinstance(r[0]._engine, FastSequentialEngine) and r[0]._engine._launches_per_step == 10
                   for r in (sparse, cat))
        same = (sparse[1] == cat[1] and sparse[2] == cat[2]
                and torch.equal(sparse[0]._engine.fused.flat_params.view(torch.int16),
                                cat[0]._engine.fused.flat_params.view(torch.int16))
                and torch.equal(sparse[0]._engine.fused.master, cat[0]._engine.fused.master))
        sync = params_in_sync(cat[0]._engine.fused.flat_params)
        good = fast and same and sync
        print(f"[{'PASS' if good else 'FAIL'}] rank {rank}/{world} {name}: fast path {fast}, same bits as sparse "
              f"{same}, in sync {sync}, last loss {cat[1][-1]:.5f}", flush=True)
        ok = ok and good
        dist.barrier()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("CATEGORICAL HEAD CHECK", "OK" if flag.item() else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if flag.item() else 1


if __name__ == "__main__":
    sys.exit(main())
