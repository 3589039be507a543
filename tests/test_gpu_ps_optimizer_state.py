"""The parameter servers' optimizer slots in checkpoints on the HBM plane (estimator/ps_hbm.py), on one H100: a local
buffer stands in for the ps rank's shard, as in test_gpu_ps_kernels.py.  Six steps straight through must end bit for
bit where three steps, an export, a fresh shard and connection with the import, and three more steps end: masters,
every slot and the bf16 shadows.  State exported by the shared-memory plane imports into the HBM plane unchanged.
With two GPUs or more, a whole job through run_on_yarn stops at step 3 and resumes from the checkpoint."""
import copy
import os
from types import SimpleNamespace

import pytest
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import canned, ps, ps_hbm
from tf_yarn_b200.models import wide_deep as wdm
from tf_yarn_b200.parallel.symm import _RawCudaMemory

pytestmark = pytest.mark.gpu

V, B, N_CAT, N_NUM = 40, 256, 3, 5
DEEP = {"adagrad": lambda: keras.optimizers.Adagrad(0.05), "adam": lambda: keras.optimizers.Adam(0.01)}


def _net():
    torch.manual_seed(0)
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=N_CAT, n_num=N_NUM)
    return canned._WideDeepNet(wide, deep, [64, 32], 1)


def _layout(net, deep, n_ps=1):
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001, l2_regularization_strength=0.01)
    return ps.make_layout(named, n_ps, DEEP[deep](), {n: ftrl for n, _ in named if n.startswith("linear.")})


class _Hbm:
    """An HbmConnection over a fresh local region, initialised as connect_worker's chief does: masters from the
    network, slots from `ps_state` (None: fresh), shadows refreshed, global step set, kernels installed."""

    def __init__(self, tmp_path, tag, net, layout, ps_state=None, step=0):
        named = ps._named_trainables(net)
        self.region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
        comm = SimpleNamespace(arena=SimpleNamespace(peer_base={0: self.region.data_ptr()}), device=0)
        self.header = ps.ShmShard(str(tmp_path / f"header_{tag}"), 8, create=True)
        self.conn = ps_hbm.HbmConnection(layout, comm, {"ps:0": 0}, 0, [n for n, _ in named], self.header, net)
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                self.conn.remote_tensor(i).copy_(p.detach().reshape(-1).float())
            ps.init_slots(layout, self.conn.remote_tensor, ps_state)
        self.conn.refresh_shadows()
        self.header.set_global_step(step)
        self.conn.install(net)
        assert self.conn.fused_first and self.conn.fused_wide
        self.net = net

    def train(self, batches):
        for feats, y in batches:
            self.conn.refresh_adam_scale()              # what the estimator's step does first
            f = {k: v.cuda() for k, v in feats.items()}
            self.conn.pull(self.net)
            self.net.zero_grad()
            out = self.net(f).float()
            torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y.cuda().float()).backward()
            self.conn.push(self.net)
            self.conn.increment_global_step()
        torch.cuda.synchronize()

    def shadow(self, i):
        """The bf16 shadow of a remote-GEMM weight [rows, cols] (pad columns dropped)."""
        rows, cols = self.conn.layout.variables[i][1]
        ld = self.conn.shadow_ld(i)
        mem = _RawCudaMemory(self.conn.shadow_ptr(i), 2 * rows * ld, self)
        return torch.as_tensor(mem, device="cuda").view(torch.bfloat16).view(rows, ld)[:, :cols].clone()

    def values(self):
        """{name/slot: fp32 master or slot}, {name: bf16 shadow}."""
        lay = self.conn.layout
        fp32 = {f"{n}/{s}": self.conn.remote_tensor(i, s).clone() for i, (n, _) in enumerate(lay.variables)
                for s in range(1 + lay.var_slots[i])}
        return fp32, {lay.variables[i][0]: self.shadow(i) for i in self.conn.gemm}

    def close(self):
        self.header.unlink()


def _assert_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), (k, (a[k].float() - b[k].float()).abs().max().item())


@pytest.mark.parametrize("deep", ["adagrad", "adam"])
def test_hbm_plane_resumes_bit_for_bit_from_exported_slots(tmp_path, deep):
    """FTRL on the wide tower, Adagrad or Adam on the deep tower, K5 and the fused wide tower on."""
    batches = wdm.synthetic_batches(B, 6, vocab=V, seed=1, n_cat=N_CAT, n_num=N_NUM)    # V = 40: heavy duplicates
    base = _net()
    layout = _layout(base, deep)
    assert set(layout.kinds) == {"ftrl", deep}
    opened = []
    try:
        straight = _Hbm(tmp_path, "straight", copy.deepcopy(base).cuda(), layout)
        opened.append(straight)
        straight.train(batches)

        first = _Hbm(tmp_path, "first", copy.deepcopy(base).cuda(), layout)
        opened.append(first)
        first.train(batches[:3])
        weights = first.conn.state_dict_from_ps(first.net)
        state = first.conn.optimizer_state()
        assert all(t.device.type == "cpu" and t.dtype == torch.float32 for e in state.values() for t in e["slots"])

        net = copy.deepcopy(base).cuda()
        net.load_state_dict(weights)
        second = _Hbm(tmp_path, "second", net, layout, ps_state=state, step=first.conn.global_step())
        opened.append(second)
        _assert_equal(first.values()[0], second.values()[0])              # the import is exact before any step
        second.train(batches[3:])

        fp32, shadows = straight.values()
        got_fp32, got_shadows = second.values()
        _assert_equal(fp32, got_fp32)
        _assert_equal(shadows, got_shadows)
        assert second.conn.global_step() == straight.conn.global_step() == 6
    finally:
        for h in opened:
            h.close()


@pytest.mark.parametrize("deep", ["adagrad", "adam"])
def test_shared_memory_plane_state_imports_into_the_hbm_plane(tmp_path, deep):
    """Three steps on the shared-memory plane over 2 ps shards, then its weights and slots into the HBM plane over 1:
    identical fp32 masters and slots, and shadows equal to bf16(master)."""
    base = _net()
    net_cpu = copy.deepcopy(base)
    named = ps._named_trainables(net_cpu)
    lay_cpu = _layout(net_cpu, deep, n_ps=2)
    shards = [ps.ShmShard(str(tmp_path / f"shard{i}"), lay_cpu.shard_elems[i], create=True) for i in range(2)]
    hbm = None
    try:
        cpu = ps.WorkerConnection(lay_cpu, shards, [n for n, _ in named])
        for s in shards:
            s.data.zero_()
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                cpu._region(i).copy_(p.detach().reshape(-1))
        ps.init_slots(lay_cpu, cpu._region)
        shards[0].set_global_step(0)
        for feats, y in wdm.synthetic_batches(B, 3, vocab=V, seed=2, n_cat=N_CAT, n_num=N_NUM):
            cpu.pull(net_cpu)
            net_cpu.zero_grad()
            torch.nn.functional.binary_cross_entropy_with_logits(net_cpu(feats)[:, 0], y.float()).backward()
            cpu.push(net_cpu)
            cpu.increment_global_step()
        weights, state = cpu.state_dict_from_ps(net_cpu), cpu.optimizer_state()

        net = copy.deepcopy(base).cuda()
        net.load_state_dict(weights)
        hbm = _Hbm(tmp_path, "hbm", net, _layout(net, deep), ps_state=state, step=3)
        fp32, shadows = hbm.values()
        want = {f"{n}/{s}": cpu._region(i, s).cuda() for i, (n, _) in enumerate(lay_cpu.variables)
                for s in range(1 + lay_cpu.var_slots[i])}
        for i, (n, _) in enumerate(lay_cpu.variables):                             # trained slots, not fresh ones
            assert torch.any(want[f"{n}/1"] != (0.1 if lay_cpu.kinds[i] in ("adagrad", "ftrl") else 0.0)), n
        _assert_equal(want, fp32)
        assert shadows
        _assert_equal({n: hbm.conn.remote_tensor(i).view(hbm.conn.layout.variables[i][1]).to(torch.bfloat16)
                       for i, (n, _) in enumerate(hbm.conn.layout.variables) if i in hbm.conn.gemm}, shadows)
    finally:
        if hbm is not None:
            hbm.close()
        for s in shards:
            s.unlink()


@pytest.mark.slow
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("deep", ["adagrad", "adam"])
def test_hbm_plane_job_resumes_bit_for_bit(tmp_path, deep):
    """test_ps_optimizer_state.py's resumed job through the HBM plane: chief and ps on their own GPUs.  One trainer's
    step is deterministic, so the resumed job ends where the uninterrupted one does, bit for bit."""
    from test_ps_optimizer_state import _assert_same, _ckpt, _train
    straight, resumed = tmp_path / "straight", tmp_path / "resumed"
    _train(straight, deep, gpu=True)
    _train(resumed, deep, max_steps=3, gpu=True)
    _train(resumed, deep, gpu=True)
    a = _ckpt(straight, 6)
    assert os.path.exists(os.path.join(str(resumed), "model.ckpt-3"))
    _assert_same(a, _ckpt(resumed, 6))
    assert {e["kind"] for e in a["ps_state"].values()} == {"ftrl", deep}
