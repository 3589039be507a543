"""PytorchExperiment: LeNet-style CIFAR-10 network, data-parallel over 2 workers x 2 processes.

(reference: tf_yarn/examples/pytorch/pytorch_example.py:19-108)

``main_fn`` receives the model wrapped for data-parallel training: on H100 that wrapper reduces the
gradient buckets with the NVLS all-reduce kernels while backward is still running.
CIFAR-10 is not downloadable on an air-gapped box: a synthetic dataset of the same shape is used.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch
import torch.nn as nn
import torch.nn.functional as F

from tf_yarn_b200.pytorch import (DataLoaderArgs, NodeLabel, PytorchExperiment, TaskSpec, model_ckpt, run_on_yarn)

logging.basicConfig(level="INFO")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"pytorch_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 6, 5)
        self.pool = nn.MaxPool2d(2, 2)
        self.conv2 = nn.Conv2d(6, 16, 5)
        self.fc1 = nn.Linear(16 * 5 * 5, 120)
        self.fc2 = nn.Linear(120, 84)
        self.fc3 = nn.Linear(84, 10)

    def forward(self, x):
        x = self.pool(F.relu(self.conv1(x)))
        x = self.pool(F.relu(self.conv2(x)))
        x = torch.flatten(x, 1)
        x = F.relu(self.fc1(x))
        x = F.relu(self.fc2(x))
        return self.fc3(x)


def main_fn(model, trainloader, device, rank, tb_writer):
    criterion = nn.CrossEntropyLoss()
    optimizer = torch.optim.SGD(model.parameters(), lr=0.001, momentum=0.9)
    for epoch in range(int(os.environ.get("EXAMPLE_EPOCHS", "2"))):
        if hasattr(trainloader, "sampler") and hasattr(trainloader.sampler, "set_epoch"):
            trainloader.sampler.set_epoch(epoch)
        running_loss = 0.0
        for i, (inputs, labels) in enumerate(trainloader):
            inputs, labels = inputs.to(device), labels.to(device)
            optimizer.zero_grad()
            loss = criterion(model(inputs), labels)
            loss.backward()
            optimizer.step()
            running_loss += loss.item()
            if i % 50 == 49:
                tb_writer.add_scalar("loss", running_loss / 50, epoch * len(trainloader) + i)
                running_loss = 0.0
        if rank == 0:
            model_ckpt.save_ckpt(MODEL_DIR, model, optimizer, epoch)


def experiment_fn() -> PytorchExperiment:
    g = torch.Generator().manual_seed(0)
    trainset = torch.utils.data.TensorDataset(torch.randn(2048, 3, 32, 32, generator=g),
                                              torch.randint(0, 10, (2048,), generator=g))
    return PytorchExperiment(model=Net(), main_fn=main_fn, train_dataset=trainset,
                             dataloader_args=DataLoaderArgs(batch_size=4, num_workers=0, shuffle=True),
                             tensorboard_hdfs_dir=os.path.join(MODEL_DIR, "tensorboard"))


def main():
    return run_on_yarn(experiment_fn, task_specs={
        "worker": TaskSpec(memory="4 GiB", vcores=4, instances=2, nb_proc_per_worker=2, label=LABEL)})


if __name__ == "__main__":
    print(main())
