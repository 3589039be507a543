"""Asynchronous parameter-server data plane for the Estimator facade.

TF's PS strategy (what the reference's default task sets up through ``TF_CONFIG``
+ ``tf.distribute.Server``; reference: tf_yarn/tensorflow/cluster.py:41-67,
tf_yarn/tensorflow/tasks/tf_task_common.py:46-50) places every variable on a
``ps`` task (round-robin), workers pull the values they need before a step and
push gradients after it; the ps applies them WITHOUT any barrier between
workers (``use_locking=False``: hogwild).

Here a ps task owns a *shard*: one flat fp32 region holding its variables and
their optimizer slots.  There is no server thread on the data path -- workers
read (pull) and update (push) the shard memory directly:

* CPU box (plumbing / CI):  the shard is a POSIX shared-memory file mapped by
  every worker (``ShmShard``).
* H100:  the shard lives in the ps rank's HBM inside the symmetric arena;
  workers reach it over NVLink with the K5 (pull) / K6 (push) kernels
  (``HbmShard``, :mod:`tf_yarn_b200.parallel.ps_kernels`).

Control (layout, readiness, global step) goes through the launcher's KV store
and a tiny shared-memory header.
"""
from __future__ import annotations

import fcntl
import json
import logging
import mmap
import os
import struct
import time
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from tf_yarn_b200 import _task_commons

logger = logging.getLogger(__name__)

KV_LAYOUT = "ps/layout"
KV_READY = "ps/ready"

# optimizer slots per variable (besides the value itself), in their order in the shard
_SLOT_NAMES = {"sgd": (), "adagrad": ("accumulator",), "adadelta": ("accum_grad", "accum_update"), "adam": ("m", "v"),
               "adamw": ("m", "v"), "ftrl": ("n", "z"), "adamax": ("m", "u")}


def slot_names(kind: str, hyper: Dict[str, float]) -> Tuple[str, ...]:
    """Slots of one variable, in shard order.  RMSprop's depend on its hyper-parameters: mean square, then the
    momentum buffer (p2 = momentum > 0), then the mean gradient (flags bit 0 = centered)."""
    if kind == "rmsprop":
        return ("ms",) + (("momentum",) if hyper["p2"] > 0 else ()) + (("mg",) if int(hyper["flags"]) & 1 else ())
    return _SLOT_NAMES[kind]


def _var_slots(kind: str, hyper: Dict[str, float]) -> int:
    return len(slot_names(kind, hyper))


def _job_tag() -> str:
    return f"{os.environ.get('TFY_APP_ID', 'local')}_{_task_commons.n_try()}"


def _shm_dir() -> str:
    return "/dev/shm" if os.path.isdir("/dev/shm") else "/tmp"


class Layout:
    """Where every variable lives: owner ps, offset inside the owner's shard."""

    def __init__(self, variables: List[Tuple[str, List[int]]], n_ps: int, opt_kind: str, hyper: Dict[str, float],
                 kinds: Optional[List[str]] = None, hypers: Optional[List[Dict[str, float]]] = None):
        self.variables = variables
        self.n_ps = n_ps
        self.opt_kind = opt_kind          # default optimizer; `kinds[i]` / `hypers[i]` are per variable
        self.hyper = hyper
        self.kinds = list(kinds) if kinds else [opt_kind] * len(variables)
        self.hypers = list(hypers) if hypers else [hyper] * len(variables)
        self.var_slots = [_var_slots(k, h) for k, h in zip(self.kinds, self.hypers)]
        self.slots = max(self.var_slots + [0])
        self.owner: List[int] = []
        self.offset: List[int] = []
        self.numel: List[int] = []
        self.shard_elems = [0] * n_ps
        for i, (_, shape) in enumerate(variables):
            n = int(np.prod(shape)) if shape else 1
            n_pad = (n + 7) // 8 * 8
            ps = i % n_ps                      # round-robin placement, like TF's default device setter
            self.owner.append(ps)
            self.offset.append(self.shard_elems[ps])
            self.numel.append(n)
            self.shard_elems[ps] += n_pad * (1 + self.var_slots[i])

    def padded(self, i: int) -> int:
        return (self.numel[i] + 7) // 8 * 8

    def to_json(self) -> str:
        return json.dumps({"variables": self.variables, "n_ps": self.n_ps, "opt_kind": self.opt_kind,
                           "hyper": self.hyper, "kinds": self.kinds, "hypers": self.hypers})

    @classmethod
    def from_json(cls, raw) -> "Layout":
        d = json.loads(raw.decode() if isinstance(raw, (bytes, bytearray)) else raw)
        return cls([(n, list(s)) for n, s in d["variables"]], d["n_ps"], d["opt_kind"], d["hyper"], d.get("kinds"),
                   d.get("hypers"))


HEADER_BYTES = 64   # [0:8] global step (int64, only meaningful on ps 0)


class ShmShard:
    """One ps task's shard as a shared-memory file: header + fp32 payload."""

    def __init__(self, path: str, n_elems: int, create: bool):
        self.path = path
        nbytes = HEADER_BYTES + 4 * max(n_elems, 8)
        if create:
            fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_TRUNC, 0o600)
            os.ftruncate(fd, nbytes)
        else:
            fd = os.open(path, os.O_RDWR)
        self._fd = fd
        self._mm = mmap.mmap(fd, nbytes)
        self.data = torch.frombuffer(self._mm, dtype=torch.float32, offset=HEADER_BYTES, count=max(n_elems, 8))

    def add_global_step(self, delta: int) -> int:
        fcntl.lockf(self._fd, fcntl.LOCK_EX, 8, 0)
        try:
            (cur,) = struct.unpack_from("<q", self._mm, 0)
            cur += delta
            struct.pack_into("<q", self._mm, 0, cur)
        finally:
            fcntl.lockf(self._fd, fcntl.LOCK_UN, 8, 0)
        return cur

    def global_step(self) -> int:
        return struct.unpack_from("<q", self._mm, 0)[0]

    def set_global_step(self, v: int) -> None:
        struct.pack_into("<q", self._mm, 0, int(v))

    def unlink(self) -> None:
        try:
            os.unlink(self.path)
        except OSError:
            pass


def _hyper_of(desc) -> Dict[str, float]:
    spec = desc.to_spec()
    return {"lr": spec.lr, "p1": spec.p1, "p2": spec.p2, "eps": spec.eps, "wd": spec.weight_decay,
            "init_s1": spec.init_s1, "flags": spec.flags}


class WorkerConnection:
    """What a chief / worker holds: the mapped shards and the variable -> region table."""

    def __init__(self, layout: Layout, shards: List[ShmShard], names: List[str], schedules=None):
        self.layout, self.shards, self.names = layout, shards, names
        # per variable: the LearningRateSchedule of its optimizer (None: the layout's constant lr)
        self.schedules = list(schedules) if schedules else [None] * len(names)
        self._t = 0

    def _region(self, i: int, slot: int = 0) -> torch.Tensor:
        lay = self.layout
        base = lay.offset[i] + slot * lay.padded(i)
        return self.shards[lay.owner[i]].data[base:base + lay.numel[i]]

    # ---- pull: ps -> local replica -------------------------------------------------
    def pull(self, network: nn.Module) -> None:
        params = dict(network.named_parameters())
        with torch.no_grad():
            for i, name in enumerate(self.names):
                p = params[name]
                p.copy_(self._region(i).view(p.shape))

    # ---- push: apply the local gradients to the ps copy (no locks: hogwild) -----------
    def push(self, network: nn.Module) -> None:
        lay = self.layout
        params = dict(network.named_parameters())
        self._t += 1
        # one global step for the whole push (another worker may advance it meanwhile): the pushes applied so far
        step = max(self.global_step(), 0) if any(s is not None for s in self.schedules) else 0
        with torch.no_grad():
            for i, name in enumerate(self.names):
                g = params[name].grad
                if g is None:
                    continue
                h = lay.hypers[i]
                lr, p1, p2, eps, wd = h["lr"], h["p1"], h["p2"], h["eps"], h["wd"]
                if self.schedules[i] is not None:
                    lr = float(self.schedules[i](step))
                g = g0 = g.detach().reshape(-1).float().cpu()
                w = self._region(i)
                if wd:
                    g = g + wd * w
                kind = lay.kinds[i]
                if kind == "sgd":
                    w.add_(g, alpha=-lr)
                elif kind == "adagrad":
                    acc = self._region(i, 1)
                    acc.addcmul_(g, g)
                    w.addcdiv_(g, acc.sqrt().add_(eps), value=-lr)
                elif kind == "ftrl":           # p1 = l1, p2 = l2, eps = beta (OptimizerSpec.ftrl)
                    n, z = self._region(i, 1), self._region(i, 2)
                    n_new = n + g * g
                    z.add_(g - (n_new.sqrt() - n.sqrt()) / lr * w)
                    n.copy_(n_new)
                    neww = -(z - torch.sign(z) * p1) / ((eps + n_new.sqrt()) / lr + 2 * p2)
                    w.copy_(torch.where(z.abs() <= p1, torch.zeros_like(neww), neww))
                elif kind == "rmsprop":        # p1 = rho, p2 = momentum, flags bit 0 = centered (OptimizerSpec.rmsprop)
                    v = self._region(i, 1)
                    v.mul_(p1).addcmul_(g, g, value=1 - p1)
                    denom = v
                    if int(h["flags"]) & 1:
                        mg = self._region(i, 3 if p2 > 0 else 2)
                        mg.mul_(p1).add_(g, alpha=1 - p1)
                        denom = v - mg * mg
                    inc = lr * g * (denom + eps).rsqrt()
                    if p2 > 0:
                        m = self._region(i, 2)
                        m.mul_(p2).add_(inc)
                        w.sub_(m)
                    else:
                        w.sub_(inc)
                elif kind == "adamax":         # lazy: rows whose gradient is all zero keep their value and slots
                    rows = params[name].shape[0] if params[name].dim() > 0 else 1
                    hit = (g0.view(rows, -1) != 0).any(dim=1)
                    m, u = self._region(i, 1).view(rows, -1), self._region(i, 2).view(rows, -1)
                    gr, wr = g.view(rows, -1)[hit], w.view(rows, -1)
                    t = max(self.global_step(), 0) + 1     # the step being applied, as for Adam
                    m[hit] = p1 * m[hit] + (1 - p1) * gr
                    u[hit] = torch.maximum(p2 * u[hit], gr.abs())
                    wr[hit] = wr[hit] - lr / (1 - p1 ** t) * m[hit] / (u[hit] + eps)
                elif kind == "adadelta":
                    sq, dx = self._region(i, 1), self._region(i, 2)
                    sq.mul_(p1).addcmul_(g, g, value=1 - p1)
                    upd = g * (dx + eps).sqrt() / (sq + eps).sqrt()
                    dx.mul_(p1).addcmul_(upd, upd, value=1 - p1)
                    w.add_(upd, alpha=-lr)
                else:  # adam: bias correction from the shared global step, like the HBM plane (ps_hbm.refresh_adam_scale)
                    m, v = self._region(i, 1), self._region(i, 2)
                    m.mul_(p1).add_(g, alpha=1 - p1)
                    v.mul_(p2).addcmul_(g, g, value=1 - p2)
                    t = max(self.global_step(), 0) + 1     # the step being applied: incremented AFTER the push
                    bc1, bc2 = 1 - p1 ** t, 1 - p2 ** t
                    w.addcdiv_(m, (v / bc2).sqrt().add_(eps), value=-lr / bc1)

    # ---- global step -------------------------------------------------------------------
    def increment_global_step(self) -> int:
        return self.shards[0].add_global_step(1)

    def global_step(self) -> int:
        return self.shards[0].global_step()

    def state_dict_from_ps(self, network: nn.Module) -> Dict[str, torch.Tensor]:
        """The network's state dict with parameter values read from the ps shards."""
        self.pull(network)
        return network.state_dict()

    def optimizer_state(self) -> Dict[str, dict]:
        """Every variable's optimizer slots, read from the ps shards (`export_slots`)."""
        return export_slots(self.layout, self._region)


def _named_trainables(network: nn.Module) -> List[Tuple[str, nn.Parameter]]:
    return [(n, p) for n, p in network.named_parameters() if p.requires_grad]


def make_layout(named, n_ps: int, opt_desc, opt_by_name=None) -> Layout:
    """Layout with the optimizer (kind + hyper-parameters) of every variable."""
    descs = [(opt_by_name or {}).get(n, opt_desc) for n, _ in named]
    return Layout([(n, list(p.shape)) for n, p in named], n_ps, opt_desc.to_spec().kind, _hyper_of(opt_desc),
                  [d.to_spec().kind for d in descs], [_hyper_of(d) for d in descs])


# ---- optimizer slots in checkpoints (both data planes) ----------------------------------------------
def export_slots(layout: Layout, region) -> Dict[str, dict]:
    """A checkpoint's ``ps_state``: per variable name its optimizer kind, shape, slot names and slots (fp32 CPU
    copies, in shard order).  region(i, s) is slot s of variable i in the shards (slot 0: the value, not saved here).
    """
    out = {}
    for i, (name, shape) in enumerate(layout.variables):
        names = slot_names(layout.kinds[i], layout.hypers[i])
        out[name] = {"kind": layout.kinds[i], "shape": list(shape), "slot_names": list(names),
                     "slots": [region(i, s).detach().to(device="cpu", dtype=torch.float32, copy=True)
                               for s in range(1, 1 + len(names))]}
    return out


def match_slots(ps_state: Dict[str, dict], layout: Layout) -> List[Optional[List[torch.Tensor]]]:
    """Per variable of `layout`: the saved slots of `ps_state` to install, or None for fresh ones.  Variables are
    matched by name, so the number of ps tasks may change.  A variable's slots are restored when its optimizer kind,
    its slots and its element count all match the saved ones; hyper-parameters such as the learning rate may differ,
    as in TF.  One warning names every variable that starts fresh."""
    out: List[Optional[List[torch.Tensor]]] = []
    fresh = []
    for i, (name, _) in enumerate(layout.variables):
        e = ps_state.get(name)
        want = list(slot_names(layout.kinds[i], layout.hypers[i]))
        n = layout.numel[i]
        if e is not None and e["kind"] == layout.kinds[i] and list(e.get("slot_names", ())) == want and \
                int(np.prod(e["shape"])) == n and len(e["slots"]) == len(want) and \
                all(t.numel() == n for t in e["slots"]):
            out.append(list(e["slots"]))
        else:
            out.append(None)
            fresh.append(name)
    if fresh:
        logger.warning("parameter-server optimizer state of %s does not match the checkpoint; starting it fresh",
                       ", ".join(fresh))
    return out


def init_slots(layout: Layout, region, ps_state: Optional[Dict[str, dict]] = None) -> None:
    """The chief's initialisation of every variable's optimizer slots in zeroed shards: the slots of a checkpoint's
    `ps_state` where `match_slots` restores them, else the optimizer's initial values (Adagrad's and FTRL's first
    slot at init_s1, every other slot 0).  region(i, s) as for `export_slots`."""
    saved = match_slots(ps_state, layout) if ps_state is not None else [None] * len(layout.variables)
    for i, slots in enumerate(saved):
        if slots is not None:
            for s, t in enumerate(slots, 1):
                region(i, s).copy_(t.reshape(-1))
        elif layout.kinds[i] in ("adagrad", "ftrl"):
            region(i, 1).fill_(layout.hypers[i]["init_s1"])


def refuse_nadam(named, opt_desc, opt_by_name=None) -> None:
    """Both parameter-server planes refuse Nadam: the running product of its momentum schedule belongs to one
    optimizer, which asynchronous workers do not share."""
    for name, _ in named:
        if (opt_by_name or {}).get(name, opt_desc).to_spec().kind == "nadam":
            raise ValueError(f"the parameter server does not run Nadam (variable {name!r}): the running product of "
                             "its momentum schedule belongs to one optimizer, which asynchronous workers do not "
                             "share; use Adam")


def connect_worker(network: nn.Module, opt_desc, cluster, is_chief: bool, global_step: int,
                   opt_by_name=None, ps_state: Optional[Dict[str, dict]] = None) -> WorkerConnection:
    """Chief: publish the layout, wait for the shards, initialise them (the optimizer slots from `ps_state`, a
    checkpoint's, where they match: `init_slots`).  Worker: wait until ready."""
    named = _named_trainables(network)
    refuse_nadam(named, opt_desc, opt_by_name)
    client = _task_commons.TaskClient.from_current()
    kv = client.kv
    n_ps = len(cluster.spec["ps"])
    names = [n for n, _ in named]
    if is_chief:
        layout = make_layout(named, n_ps, opt_desc, opt_by_name)
        kv[KV_LAYOUT] = layout.to_json().encode()
    else:
        layout = Layout.from_json(kv.wait(KV_LAYOUT))
    shards = []
    for i in range(n_ps):
        path = kv.wait(f"ps:{i}/shard").decode()
        shards.append(ShmShard(path, layout.shard_elems[i], create=False))
    conn = WorkerConnection(layout, shards, names,
                            [getattr((opt_by_name or {}).get(n, opt_desc), "schedule", None) for n in names])
    if is_chief:
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                conn._region(i).copy_(p.detach().reshape(-1).float().cpu())
            init_slots(layout, conn._region, ps_state)
        shards[0].set_global_step(global_step)
        kv[KV_READY] = b"1"
        logger.info("parameter servers initialised: %d variables on %d ps", len(names), n_ps)
    else:
        kv.wait(KV_READY)
    return conn


def serve(cluster, poll_secs: float = 0.2) -> None:
    """Body of a ``ps`` task: allocate the shard, publish it, then idle (never returns).

    Like ``tf.distribute.Server.join()`` this blocks forever; the task program runs it on a
    daemon thread and leaves through the stop barrier once every trainer has stopped.
    """
    client = _task_commons.TaskClient.from_current()
    kv = client.kv
    idx = cluster.task_id
    layout = Layout.from_json(kv.wait(KV_LAYOUT))
    path = os.path.join(_shm_dir(), f"tfy_ps_{_job_tag()}_{idx}")
    shard = ShmShard(path, layout.shard_elems[idx], create=True)
    shard.data.zero_()
    kv[f"ps:{idx}/shard"] = path.encode()
    logger.info("ps %d serving %d fp32 elements from %s", idx, layout.shard_elems[idx], path)
    import atexit
    atexit.register(shard.unlink)
    while True:
        time.sleep(poll_secs)
