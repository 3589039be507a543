"""tf_yarn_b200: a H100-native distributed-training launcher with the capabilities of criteo/tf-yarn.

Public surface (reference: tf_yarn/__init__.py:1-8)::

    from tf_yarn_b200 import TaskSpec, NodeLabel, single_server_topology, ps_strategy_topology, \
        get_safe_experiment_fn, RunFailed, Metrics

Front-ends: ``tf_yarn_b200.tensorflow`` (Estimator / Keras experiments; torch-backed facades),
``tf_yarn_b200.pytorch`` (PytorchExperiment), ``tf_yarn_b200.distributed`` (any ``fn(local_rank)``).
"""
from tf_yarn_b200.client import RunFailed, get_safe_experiment_fn
from tf_yarn_b200.metrics import Metrics
from tf_yarn_b200.topologies import (NodeLabel, TaskSpec, allreduce_topology, ps_strategy_topology,
                                     single_server_topology)

__version__ = "0.2.0"

__all__ = ["get_safe_experiment_fn", "RunFailed", "Metrics", "TaskSpec", "NodeLabel", "single_server_topology",
           "ps_strategy_topology", "allreduce_topology"]
