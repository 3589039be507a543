"""An HbmConnection (estimator/ps_hbm.py) over fake ps base addresses and CPU tensors: enough for the routing
decisions it takes and, with a recording kernel library, for whole worker steps without a GPU."""
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import ps, ps_hbm

OPTIMIZERS = {"sgd": lambda: keras.optimizers.SGD(0.1), "adagrad": lambda: keras.optimizers.Adagrad(0.05),
              "adam": lambda: keras.optimizers.Adam(0.01),
              "ftrl": lambda: keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001,
                                                    l2_regularization_strength=0.01, beta=0.5)}


def hbm_connection(network, opt="adagrad", n_ps=2, by_name=None, lib=None):
    """opt names the default optimizer, by_name maps variable names to optimizer names; lib stands in for the kernel
    library (None: no kernel may be called)."""
    named = ps._named_trainables(network)
    by_name = {n: OPTIMIZERS[o]() for n, o in (by_name or {}).items()}
    layout = ps.make_layout(named, n_ps, OPTIMIZERS[opt](), by_name or None)
    conn = ps_hbm.HbmConnection.__new__(ps_hbm.HbmConnection)
    conn.layout, conn.names, conn.lib = layout, [n for n, _ in named], lib
    conn.var_opt = [ps_hbm.OPT_CODES[k] for k in layout.kinds]
    conn.ps_base = [1 << 40, 2 << 40][:n_ps] + [3 << 40] * max(0, n_ps - 2)
    conn.device = torch.device("cpu")
    params = dict(network.named_parameters())
    conn.params = [params[n] for n in conn.names]
    conn.sparse, conn.gemm = {}, {}
    conn._classify(network)
    conn.dense_idx = [i for i in range(len(conn.names)) if i not in conn.sparse]
    conn.pull_idx = [i for i in conn.dense_idx if i not in conn.gemm]
    conn._pull_segs = conn._make_segs(for_push=False, idx=conn.pull_idx)
    conn._push_segs = conn._push_ptrs = None
    conn._max_n = max([conn._n4(i) for i in conn.dense_idx] + [4])
    conn.adam_scale = torch.ones(2)
    conn._acct = {"pull_bytes": 0, "push_bytes": 0, "launches_per_step": 0}
    conn._acct_last = dict(conn._acct)
    return conn
