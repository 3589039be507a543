"""mini-Estimator: a torch-backed subset of ``tf.estimator`` (TensorFlow is not required).

Covers what the reference's task programs and examples touch (SURVEY.md appendix A):
Estimator / RunConfig / TrainSpec / EvalSpec / EstimatorSpec / ModeKeys / train_and_evaluate /
session-run hooks / checkpoint index / exporters / canned LinearClassifier, DNNClassifier,
DNNLinearCombinedClassifier, LinearRegressor, DNNRegressor, DNNLinearCombinedRegressor / heads (BinaryClassHead,
MultiClassHead, RegressionHead, MultiLabelHead, PoissonRegressionHead, LogisticRegressionHead) and the
LinearEstimator, DNNEstimator and DNNLinearCombinedEstimator that take one / feature columns / model_to_estimator.
"""
from tf_yarn_b200.estimator import feature_column  # noqa: F401
from tf_yarn_b200.estimator.canned import (SUM_OVER_BATCH_SIZE, DNNClassifier,  # noqa: F401
                                           DNNEstimator, DNNLinearCombinedClassifier, DNNLinearCombinedEstimator,
                                           DNNLinearCombinedRegressor, DNNRegressor, LinearClassifier,
                                           LinearEstimator, LinearRegressor, model_to_estimator)
from tf_yarn_b200.estimator.checkpoint import get_checkpoint_state, latest_checkpoint  # noqa: F401
from tf_yarn_b200.estimator.config import ClusterInfo, ConfigProto, RunConfig, SessionConfig  # noqa: F401
from tf_yarn_b200.estimator.estimator import Estimator  # noqa: F401
from tf_yarn_b200.estimator.exporter import BestExporter, Exporter, FinalExporter, LatestExporter  # noqa: F401
from tf_yarn_b200.estimator.head import (BinaryClassHead, LogisticRegressionHead, MultiClassHead,  # noqa: F401
                                         MultiLabelHead, PoissonRegressionHead, RegressionHead)
from tf_yarn_b200.estimator.hooks import (LoggingTensorHook, NanTensorHook, SessionRunArgs,  # noqa: F401
                                          SessionRunContext, SessionRunHook, SessionRunValues, StepCounterHook,
                                          StopAtStepHook, get_global_step)
from tf_yarn_b200.estimator.spec import EstimatorSpec, EvalSpec, GraphKeys, ModeKeys, TrainSpec  # noqa: F401
from tf_yarn_b200.estimator.training import continuous_eval, train_and_evaluate  # noqa: F401
