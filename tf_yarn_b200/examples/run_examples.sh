#!/usr/bin/env bash
# Runs every example on this box (reference: tf_yarn/examples/run_examples.sh, run_pytorch_examples.sh).
set -euo pipefail
for ex in id_estimator_example linear_classifier_example keras_example native_keras_with_gloo_example \
          collective_all_reduce_example mlflow_example pytorch.pytorch_example pytorch.pytorch_distributed_example; do
  echo "=== $ex"
  EXAMPLE_EPOCHS=1 python -m tf_yarn_b200.examples.$ex
done
# the BASELINE.json configurations (full size on H100, toy size on a CPU-only box or with EXAMPLE_SMALL=1)
for ex in baseline.mnist_cnn_allreduce baseline.wide_deep_ps baseline.resnet50_ddp baseline.bert_allreduce; do
  echo "=== $ex"
  EXAMPLE_EPOCHS=1 python -m tf_yarn_b200.examples.$ex
done
