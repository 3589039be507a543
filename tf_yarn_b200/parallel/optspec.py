"""Fused-optimizer hyper-parameter description (no CUDA dependency)."""
from __future__ import annotations

OPT_SGD, OPT_ADADELTA, OPT_ADAM, OPT_ADAGRAD, OPT_FTRL, OPT_RMSPROP, OPT_ADAMAX, OPT_NADAM = range(8)


class OptimizerSpec:
    """Hyper-parameters of a fused optimizer (device-independent description)."""

    KINDS = {"sgd": OPT_SGD, "adadelta": OPT_ADADELTA, "adam": OPT_ADAM,
             "adamw": OPT_ADAM, "adagrad": OPT_ADAGRAD, "ftrl": OPT_FTRL, "rmsprop": OPT_RMSPROP,
             "adamax": OPT_ADAMAX, "nadam": OPT_NADAM}

    def __init__(self, kind: str, lr: float, p1: float = 0.0, p2: float = 0.0, eps: float = 1e-7,
                 weight_decay: float = 0.0, flags: int = 0, init_s1: float = 0.0):
        kind = kind.lower()
        if kind not in self.KINDS:
            raise ValueError(f"unknown fused optimizer {kind!r}")
        # a learning-rate schedule (keras.optimizers.schedules): `lr` is its rate at step 0, the fused step writes the
        # rate of every later step on the device
        self.schedule = lr if callable(lr) and hasattr(lr, "get_config") else None
        if self.schedule is not None:
            lr = self.schedule(0)
        self.kind, self.lr, self.p1, self.p2, self.eps = kind, float(lr), float(p1), float(p2), float(eps)
        self.weight_decay, self.flags, self.init_s1 = float(weight_decay), int(flags), float(init_s1)
        if kind == "adamw":
            self.flags |= 1

    @property
    def code(self) -> int:
        return self.KINDS[self.kind]

    @property
    def n_states(self) -> int:
        if self.kind == "rmsprop":
            return 1 + (self.p2 > 0) + (self.flags & 1)
        return 2 if self.kind in ("adadelta", "adam", "adamw", "ftrl", "adamax", "nadam") else 1

    def s2_numel(self, shard_n: int) -> int:
        """Length of the fp32 ``s2`` buffer of a shard of ``shard_n`` elements: every state after the first, back to
        back (at least 8 elements, so the kernel always gets a valid pointer)."""
        return max(8, shard_n * (self.n_states - 1))

    @staticmethod
    def sgd(lr, momentum=0.0, dampening=0.0, nesterov=False, weight_decay=0.0):
        return OptimizerSpec("sgd", lr, momentum, dampening, 0.0, weight_decay, 1 if nesterov else 0)

    @staticmethod
    def adadelta(lr=1.0, rho=0.95, eps=1e-7, weight_decay=0.0):
        return OptimizerSpec("adadelta", lr, rho, 0.0, eps, weight_decay)

    @staticmethod
    def adam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, decoupled=False):
        return OptimizerSpec("adamw" if decoupled else "adam", lr, beta1, beta2, eps, weight_decay)

    @staticmethod
    def adagrad(lr=1e-2, eps=1e-10, weight_decay=0.0, initial_accumulator_value=0.0):
        return OptimizerSpec("adagrad", lr, 0.0, 0.0, eps, weight_decay, init_s1=initial_accumulator_value)

    @staticmethod
    def ftrl(lr=1e-3, l1=0.0, l2=0.0, beta=0.0, initial_accumulator_value=0.1, weight_decay=0.0):
        """FTRL-proximal with learning_rate_power = -0.5 (TF's FtrlOptimizer default): s1 = accumulator n
        (initial_accumulator_value), s2 = linear z; p1 = l1, p2 = l2, eps carries beta."""
        return OptimizerSpec("ftrl", lr, l1, l2, beta, weight_decay, init_s1=initial_accumulator_value)

    @staticmethod
    def rmsprop(lr=1e-3, rho=0.9, momentum=0.0, eps=1e-7, centered=False, weight_decay=0.0):
        """RMSprop as tf.keras defines it (epsilon inside the square root, lr inside the momentum buffer): s1 = mean
        square; s2 = momentum buffer (momentum > 0) then mean gradient (centered), each shard long; p1 = rho,
        p2 = momentum, flags bit 0 = centered."""
        if momentum < 0:
            raise ValueError(f"RMSprop momentum must be >= 0, got {momentum}")
        return OptimizerSpec("rmsprop", lr, rho, momentum, eps, weight_decay, 1 if centered else 0)

    @staticmethod
    def adamax(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7, weight_decay=0.0):
        """Adamax as tf.keras defines it: s1 = m, s2 = u = max(beta2 u, |g|), p -= lr / (1 - beta1^t) m / (u + eps)
        (epsilon outside the max); p1 = beta1, p2 = beta2."""
        return OptimizerSpec("adamax", lr, beta1, beta2, eps, weight_decay)

    @staticmethod
    def nadam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7, weight_decay=0.0):
        """Nadam as torch.optim.NAdam with momentum_decay = 0.004 (tf.keras 2's schedule_decay): s1 = m, s2 = v;
        p1 = beta1, p2 = beta2.  The running product of its momentum schedule follows the hyper-parameters on the
        device (TfyNadamHyperBlock)."""
        return OptimizerSpec("nadam", lr, beta1, beta2, eps, weight_decay)
