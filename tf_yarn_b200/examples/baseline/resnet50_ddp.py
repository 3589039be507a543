"""BASELINE config 4: PytorchExperiment ResNet-50 under DistributedDataParallel, one worker per H100.

    python -m tf_yarn_b200.examples.baseline.resnet50_ddp

The user code is what the reference expects (reference: tf_yarn/pytorch/experiment.py:6-56,
examples/pytorch/pytorch_example.py:39-108): ``main_fn(model, loader, device, rank, tb_writer)`` receives the model
already wrapped.  On H100 the wrapper is this repo's (bucketed NVLS reduction launched by a native reducer while
backward runs); ``model.fuse_optimizer("sgd", ...)`` additionally moves the optimizer into that exchange.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch
import torch.nn as nn

from tf_yarn_b200.examples import baseline
from tf_yarn_b200.pytorch import (DataLoaderArgs, DistributedDataParallelArgs, NodeLabel, PytorchExperiment, TaskSpec,
                                  model_ckpt, run_on_yarn)

logging.basicConfig(level="INFO")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"resnet50_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU
SMALL = baseline.small()
N_IMAGES, SIDE, BATCH = (64, 32, 8) if SMALL else (int(os.environ.get("EXAMPLE_IMAGES", "4096")), 224, 64)


class SyntheticImages(torch.utils.data.Dataset):
    def __init__(self, n: int, side: int, classes: int):
        g = torch.Generator().manual_seed(0)
        self.x = torch.randn(n, 3, side, side, generator=g)
        self.y = torch.randint(0, classes, (n,), generator=g)

    def __len__(self):
        return len(self.y)

    def __getitem__(self, i):
        return self.x[i], self.y[i]


def build_model() -> nn.Module:
    if SMALL:
        return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ReLU(), nn.AdaptiveAvgPool2d(1),
                             nn.Flatten(), nn.Linear(8, 10))
    import torchvision
    return torchvision.models.resnet50()


def main_fn(model, loader, device, rank, tb_writer):
    on_gpu = str(device).startswith("cuda")
    if on_gpu and hasattr(model, "fuse_optimizer"):
        optimizer = model.fuse_optimizer("sgd", lr=0.01, momentum=0.9)        # update inside the gradient exchange
    else:
        optimizer = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    criterion = nn.CrossEntropyLoss()
    for epoch in range(int(os.environ.get("EXAMPLE_EPOCHS", "1"))):
        if hasattr(loader, "sampler") and hasattr(loader.sampler, "set_epoch"):
            loader.sampler.set_epoch(epoch)
        for step, (x, y) in enumerate(loader):
            x, y = x.to(device, non_blocking=True), y.to(device, non_blocking=True)
            optimizer.zero_grad()
            with torch.autocast("cuda" if on_gpu else "cpu", dtype=torch.bfloat16):
                loss = criterion(model(x), y)
            loss.backward()
            optimizer.step()
            if step % 20 == 0:
                tb_writer.add_scalar("loss", float(loss), epoch * len(loader) + step)
        if rank == 0:
            model_ckpt.save_ckpt(MODEL_DIR, model, optimizer, epoch)


def experiment_fn() -> PytorchExperiment:
    model = build_model()
    if torch.cuda.is_available():
        model = model.to(memory_format=torch.channels_last)
    return PytorchExperiment(model=model, main_fn=main_fn,
                             train_dataset=SyntheticImages(N_IMAGES, SIDE, 10 if SMALL else 1000),
                             dataloader_args=DataLoaderArgs(batch_size=BATCH, num_workers=0, pin_memory=True),
                             tensorboard_hdfs_dir=os.path.join(MODEL_DIR, "tensorboard"),
                             ddp_args=DistributedDataParallelArgs(bucket_cap_mb=25))


def main():
    n = baseline.n_trainers()
    return run_on_yarn(experiment_fn, {"worker": TaskSpec("16 GiB", 8, instances=n, label=LABEL)})


if __name__ == "__main__":
    print(main())
