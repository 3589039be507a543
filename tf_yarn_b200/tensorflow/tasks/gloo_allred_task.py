"""Name kept from the reference (``custom_task_module="...tasks.gloo_allred_task"``): the all-reduce
task.  The transport is NVLink on H100 and gloo only on CPU-only boxes; see :mod:`.allred_task`."""
from tf_yarn_b200.tensorflow.tasks.allred_task import *  # noqa: F401,F403
from tf_yarn_b200.tensorflow.tasks.allred_task import _driver_fn, _worker_fn, main  # noqa: F401

if __name__ == "__main__":
    main()
