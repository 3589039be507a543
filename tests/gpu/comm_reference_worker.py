"""Drive the collective kernels and the multi-GPU fused optimizer step for tests/test_gpu_comm_reference.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/gpu/comm_reference_worker.py OUT_DIR

One process per GPU.  The control plane is gloo, so the project's kernels are the only collectives on the GPUs.  This
script only launches kernels and saves what they left: rank 0's outputs (``OUT_DIR/*.npy``, ``OUT_DIR/step/*.npz``),
every rank's SHA-256 of each output (``OUT_DIR/rank<r>.json``) and the fused steps' per-rank states.  All judging
happens in the test, against tests/comm_reference.py.

The grid barriers of these kernels wait for every rank, so no rank may skip a launch the others make: every input is
built before the first launch, the script makes the same launches in the same order on every rank whatever the
results, it never asserts between launches, and every launch uses the host's own grid or a smaller one.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import comm_reference as cr  # noqa: E402
import fused_step_reference as fref  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402
from tf_yarn_b200.parallel.comm import _DT, Communicator, FusedShardedOptimizer, OptimizerSpec, launch_code  # noqa: E402
from tf_yarn_b200.parallel.symm import SoloRendezvous, StoreRendezvous, SymmArena  # noqa: E402

TDT = {"bf16": torch.bfloat16, "f32": torch.float32}
ALGO = {"oneshot": native.ALGO_ONESHOT, "twoshot": native.ALGO_TWOSHOT, "nvls": native.ALGO_NVLS}


def _np_bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().contiguous()
    if t.element_size() == 2:
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    if t.element_size() == 8:
        return t.view(torch.int64).cpu().numpy().view(np.uint64)
    return t.view(torch.int32).cpu().numpy().view(np.uint32)


def spec_of(c) -> OptimizerSpec:
    kind, hp, init = fref.VARIANTS[c.variant]
    lr = hp["lr"]
    if c.sched:
        from tf_yarn_b200.keras import schedules
        cls, kw = cr.SCHEDULES[c.variant]
        lr = getattr(schedules, cls)(**kw)
    return OptimizerSpec(kind, lr, hp.get("p1", 0.0), hp.get("p2", 0.0), hp.get("eps", 0.0), hp.get("wd", 0.0),
                         hp.get("flags", 0), init)


def _sha_t(t: torch.Tensor) -> str:
    return cr.sha(_np_bits(t).view(np.uint8)) if t.numel() else cr.sha(np.zeros(0, np.uint8))


class Worker:
    def __init__(self, out_dir: str):
        self.out = out_dir
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(self.local)
        self.dev = torch.device(f"cuda:{self.local}")
        store = dist.distributed_c10d._get_default_store()
        rdv = StoreRendezvous(store, self.rank, self.world, prefix="comm_reference")
        self.arena = SymmArena(cr.ARENA_BYTES + cr.FUSION_BYTES + (1 << 20), device=self.local, rdv=rdv)
        self.comm = Communicator(fusion_bytes=cr.FUSION_BYTES, arena=self.arena)
        self.lib = self.comm.lib
        self.ctx = self.arena.ctx_ref
        self.mc = bool(self.comm.multicast)
        self.rec = {"rank": self.rank, "world": self.world, "multicast": self.mc}
        self.stream = torch.cuda.current_stream().cuda_stream
        rb = cr.region_bytes(self.world)
        self.regions = {k: self.arena.alloc(v, align=4096) for k, v in rb.items()}
        self.region_len = rb

    # -- guarded buffers ------------------------------------------------------------------------------------------
    def _u8(self, off, nbytes):
        return self.arena.tensor(off, (nbytes,), torch.uint8)

    def _arm(self, region: str, nbytes: int, content: np.ndarray):
        """Fill the guard bands of ``region`` with this rank's sentinel and its buffer with ``content``; return the
        buffer's arena offset."""
        base = self.regions[region]
        lo, _ = cr.guarded(nbytes)
        sent = torch.from_numpy(cr.sentinel(cr.GUARD, self.rank)).to(self.dev)
        self._u8(base, cr.GUARD).copy_(sent)
        self._u8(base + lo + cr._up(nbytes, 16), cr.GUARD).copy_(sent)
        self._u8(base + lo, nbytes).copy_(torch.from_numpy(np.ascontiguousarray(content).view(np.uint8)).to(self.dev))
        return base + lo

    def _guards(self, region: str, nbytes: int):
        base = self.regions[region]
        lo, _ = cr.guarded(nbytes)
        return [_sha_t(self._u8(base, cr.GUARD)), _sha_t(self._u8(base + lo + cr._up(nbytes, 16), cr.GUARD))]

    def _save(self, name: str, arr: np.ndarray):
        if self.rank == 0:
            np.save(os.path.join(self.out, name + ".npy"), arr)

    # -- K1 / K2 / K3 ---------------------------------------------------------------------------------------------
    def allreduce(self):
        W = self.world
        inputs = {}
        for c in cr.CASES:          # every input before the first launch
            key = (c.input_key, c.algo == "oneshot")
            if key not in inputs:
                inputs[key] = cr.to_bits(cr.case_input(c, W, self.rank), c.dtype)
        out = {}
        for c in cr.CASES:
            if c.algo == "nvls" and not self.mc:
                continue
            bits = inputs[(c.input_key, c.algo == "oneshot")]
            n = bits.size
            nbytes = n * cr.ESIZE[c.dtype]
            s = cr.size_of(c, W)
            off = self._arm("ar", nbytes, bits)
            out_off = self._arm("out", nbytes, cr.junk(nbytes, self.rank, c.id))
            outp = self.arena.base + out_off if c.algo == "oneshot" else None
            torch.cuda.synchronize()
            rc = self.lib.tfy_allreduce(self.ctx, native.BF16 if c.dtype == "bf16" else native.F32, ALGO[c.algo],
                                        off, n, cr.scale_value(c.scale, W), outp, s.grid, s.block, self.stream)
            torch.cuda.synchronize()
            res = self._u8(out_off if c.algo == "oneshot" else off, nbytes).view(TDT[c.dtype])
            res_bits = _np_bits(res)
            self._save(f"ar_{c.id}", res_bits)
            out[c.id] = {"rc": int(rc), "out": cr.sha(res_bits),
                         "input_after": _sha_t(self._u8(off, nbytes)),
                         "guards": self._guards("ar", nbytes) + self._guards("out", nbytes)}
        self.rec["allreduce"] = out

    def refusals(self):
        """The launchers' host-side checks, made before any launch and the same on every rank."""
        W, off = self.world, self.regions["ar"] + cr.GUARD
        outp = self.arena.base + self.regions["out"] + cr.GUARD
        r = {"bad_n": int(self.lib.tfy_allreduce(self.ctx, native.BF16, native.ALGO_TWOSHOT, off, 8 * W + 1, 1.0,
                                                 None, 0, 0, self.stream)),
             "oneshot_no_out": int(self.lib.tfy_allreduce(self.ctx, native.F32, native.ALGO_ONESHOT, off, 4 * W, 1.0,
                                                          None, 0, 0, self.stream)),
             "bcast_bad_bytes": int(self.lib.tfy_broadcast(self.ctx, off, 17, 0, 0, 0, 0, self.stream)),
             "gather_bad_bytes": int(self.lib.tfy_allgather(self.ctx, off, 17, 0, 0, self.stream))}
        if W > 1:
            r["shard_not_divisible"] = int(self.lib.tfy_allreduce(self.ctx, native.BF16, native.ALGO_TWOSHOT, off,
                                                                  8 * (W + 1), 1.0, outp, 0, 0, self.stream))
        if not self.mc:
            r["nvls_without_multicast"] = int(self.lib.tfy_allreduce(self.ctx, native.F32, native.ALGO_NVLS, off,
                                                                     4 * W, 1.0, None, 0, 0, self.stream))
        torch.cuda.synchronize()
        self.rec["refusals"] = r

    # -- K7 broadcast and the all-gather --------------------------------------------------------------------------
    def broadcast_gather(self):
        W = self.world
        modes = [0, 1] if self.mc else [0]
        bc = {}
        for packs in cr.BCAST_PACKS:
            nb = packs * 16
            for root in range(W):
                for nvls in modes:
                    key = f"{packs}-{root}-{nvls}"
                    mine = cr.payload(nb, f"bcast-{packs}", root) if self.rank == root else cr.junk(nb, self.rank, key)
                    off = self._arm("bcast", nb, mine)
                    torch.cuda.synchronize()
                    rc = self.lib.tfy_broadcast(self.ctx, off, nb, root, nvls, 0, 0, self.stream)
                    torch.cuda.synchronize()
                    bc[key] = {"rc": int(rc), "out": _sha_t(self._u8(off, nb)), "guards": self._guards("bcast", nb)}
        ga = {}
        for packs in cr.GATHER_PACKS:
            nb = packs * 16
            buf = np.concatenate([cr.payload(nb, f"gather-{packs}", r) if r == self.rank
                                  else cr.junk(nb, self.rank, f"gather-{packs}-{r}") for r in range(W)])
            off = self._arm("gather", nb * W, buf)
            torch.cuda.synchronize()
            rc = self.lib.tfy_allgather(self.ctx, off, nb, 0, 0, self.stream)
            torch.cuda.synchronize()
            ga[str(packs)] = {"rc": int(rc), "out": _sha_t(self._u8(off, nb * W)),
                              "guards": self._guards("gather", nb * W)}
        self.rec["broadcast"], self.rec["allgather"] = bc, ga

    # -- the Communicator's list API ------------------------------------------------------------------------------
    def _list(self, rank: int, tag: str):
        """The mixed tensor list of tests/comm_reference.list_values, on the device."""
        out = []
        for name, dtype, shape, strided in cr.LIST_TENSORS:
            v = cr.list_values(name, dtype, shape, rank, tag)
            t = torch.from_numpy(v).to(self.dev).to(TDT.get(dtype, torch.float16))
            if strided:
                base = torch.zeros(shape[0], shape[1] * 3, dtype=t.dtype, device=self.dev)
                view = base[:, ::3]
                view.copy_(t)
                t = view
            out.append(t)
        return out

    def list_api(self):
        W = self.world
        lcomm = Communicator(fusion_bytes=cr.FUSION_BYTES, arena=self.arena)
        lcomm.multicast = False          # P2P transport: rank-order sums (the NVLS kernel is judged on its own)
        res = {}
        for average in (True, False):
            ts = self._list(self.rank, "reduce")
            torch.cuda.synchronize()
            lcomm.all_reduce(ts, average=average)
            torch.cuda.synchronize()
            for (name, *_), t in zip(cr.LIST_TENSORS, ts):
                b = _np_bits(t) if t.numel() else np.zeros(0, np.uint8)
                self._save(f"list_{average}_{name}", b)
                res[f"reduce-{average}-{name}"] = {"out": cr.sha(b.view(np.uint8)), "shape": list(t.shape),
                                                   "dtype": str(t.dtype)}
        root = W - 1
        ts = self._list(self.rank, "bcast")
        torch.cuda.synchronize()
        lcomm.broadcast(ts, root=root)
        torch.cuda.synchronize()
        for (name, *_), t in zip(cr.LIST_TENSORS, ts):
            b = _np_bits(t) if t.numel() else np.zeros(0, np.uint8)
            res[f"bcast-{name}"] = {"out": cr.sha(b.view(np.uint8))}
        # float64 and int64: the dtypes the kernels do not carry
        for average in (False, True):
            f64 = torch.from_numpy(cr.wide_values(np.float64, self.rank)).to(self.dev)
            i64 = torch.from_numpy(cr.wide_values(np.int64, self.rank)).to(self.dev)
            ts = [f64] if average else [f64, i64]
            torch.cuda.synchronize()
            lcomm.all_reduce(ts, average=average)
            torch.cuda.synchronize()
            for t in ts:
                nm = f"wide_{average}_{str(t.dtype)[6:]}"
                b = _np_bits(t)
                self._save(nm, b)
                res[nm] = {"out": cr.sha(b.view(np.uint8))}
        self.rec["list"] = res

    # -- K4 -------------------------------------------------------------------------------------------------------
    def fused_steps(self):
        W, R = self.world, self.rank
        os.makedirs(os.path.join(self.out, "step"), exist_ok=True)
        cases = cr.step_cases(W, self.mc)
        # every input before the first launch
        grads, masters = {}, {}
        for c in cases:
            n = cr.flat_size(cr.layout_shapes(c.layout, W), W)
            for k in range(len(cr.STEP_SCALES)):
                gk = (c.layout, c.solo_grad, k)
                if gk not in grads:
                    grads[gk] = cr.case_grads(n, c, R, k)
            kind = fref.VARIANTS[c.variant][0]
            mk = (c.layout, kind == "ftrl")
            if mk not in masters:
                masters[mk] = cr.initial_master(n, c.layout, kind == "ftrl")
        fos, solo_fos = {}, {}
        solo = None
        results = {}
        for c in cases:
            kind, hp, init = fref.VARIANTS[c.variant]
            key = (c.variant, c.pair, c.layout, c.sched)
            if key not in fos:
                fos[key] = FusedShardedOptimizer(self.comm, cr.layout_shapes(c.layout, W), spec_of(c),
                                                 param_dtype=TDT[c.pair[1]], grad_dtype=TDT[c.pair[0]])
            fo = fos[key]
            mode = native.MODE_NVLS if c.mode == "nvls" else native.MODE_P2P
            p0 = masters[(c.layout, kind == "ftrl")]
            rec = self._run_step_case(c, fo, mode, p0, [grads[(c.layout, c.solo_grad, k)]
                                                        for k in range(len(cr.STEP_SCALES))])
            if c.solo_grad:
                # the same steps on one GPU, in LOCAL mode, with rank 0's gradient
                if solo is None:
                    solo = Communicator(arena_bytes=64 << 20, fusion_bytes=1 << 20, rdv=SoloRendezvous(),
                                        device=self.local)
                if key not in solo_fos:
                    solo_fos[key] = FusedShardedOptimizer(solo, cr.layout_shapes(c.layout, W), spec_of(c),
                                                          param_dtype=TDT[c.pair[1]], grad_dtype=TDT[c.pair[0]])
                sfo = solo_fos[key]
                g0 = [cr.case_grads(fo.n, c, 0, k) for k in range(len(cr.STEP_SCALES))]
                rec["local"] = self._run_local(c, sfo, p0, g0)
            results[c.id] = rec
        self.rec["step"] = results

    def _reset(self, fo, c, p0, shard_lo):
        kind, hp, init = fref.VARIANTS[c.variant]
        S = fo.shard_n
        fo.master.copy_(torch.from_numpy(p0[shard_lo:shard_lo + S].copy()))
        fo.flat_params.copy_(torch.from_numpy(p0).to(fo.param_dtype))
        fo.flat_grads.zero_()
        fo.s1.fill_(init)
        fo.s2.zero_()
        fo.set_step_count(0)
        fo.set_grad_scale(1.0)

    def _launch(self, fo, mode, piece, zero_grads):
        c = fo.comm
        args = (c.arena.ctx_ref, _DT[fo.grad_dtype], _DT[fo.param_dtype], launch_code(fo.spec), mode, fo.grad_off,
                fo.param_off, fo.shard_n, fo.master.data_ptr(), fo.s1.data_ptr(), fo.s2.data_ptr(),
                fo.hyper.data_ptr())
        how, a, b, adv = piece
        if how == "full":
            return c.lib.tfy_fused_step(*args, int(zero_grads), 0, 0, self.stream)
        if how == "range":
            return c.lib.tfy_fused_step_range(*args, 0, 0, 0, a, b, int(adv), self.stream)
        return c.lib.tfy_fused_step_shard_range(*args, 0, 0, 0, a, b, int(adv), self.stream)

    def _state(self, fo):
        return {"master": fo.master.cpu().numpy(), "s1": fo.s1.cpu().numpy(), "s2": fo.s2.cpu().numpy()}

    def _run_step_case(self, c, fo, mode, p0, grads):
        R = self.rank
        self._reset(fo, c, p0, R * fo.shard_n)
        pieces = cr.step_pieces(c.split, fo.shard_n, self.world)
        arrays, rec = {}, {"rc": [], "grads_before": [], "grads_after": [], "params": [], "step": [], "lr": []}
        for k, scale in enumerate(cr.STEP_SCALES):
            scale = float(self.world) if c.solo_grad else scale
            fo.set_grad_scale(scale)
            fo.flat_grads.copy_(torch.from_numpy(grads[k]).to(fo.grad_dtype))
            torch.cuda.synchronize()
            for nm, a in self._state(fo).items():
                arrays[f"k{k}_before_{nm}"] = a
            rec["lr"].append(float(fo.hyper[0:4].view(torch.float32).item()))
            rec["grads_before"].append(_sha_t(fo.flat_grads))
            rcs, after = [], []
            for i, piece in enumerate(pieces):
                rcs.append(int(self._launch(fo, mode, piece, c.split == "full")))
                torch.cuda.synchronize()
                for nm, a in self._state(fo).items():
                    arrays[f"k{k}_p{i}_{nm}"] = a
                after.append({"params": _sha_t(fo.flat_params), "grads": _sha_t(fo.flat_grads),
                              "step": int(fo.hyper[24:28].view(torch.int32).item())})
                if R == 0:
                    arrays[f"k{k}_p{i}_params"] = _np_bits(fo.flat_params)
            rec["rc"].append(rcs)
            rec["after"] = rec.get("after", []) + [after]
        np.savez(os.path.join(self.out, "step", f"{c.id}_r{R}.npz"), **arrays)
        return rec

    def _run_local(self, c, fo, p0, grads):
        self._reset(fo, c, p0, 0)
        out = []
        for k in range(len(cr.STEP_SCALES)):
            fo.flat_grads.copy_(torch.from_numpy(grads[k]).to(fo.grad_dtype))
            rc = self._launch(fo, native.MODE_LOCAL, ("full", 0, 0, True), True)
            torch.cuda.synchronize()
            n, S = fo.shard_n, fo.shard_n // self.world
            lo = self.rank * S
            st = {"master": _np_bits(fo.master[lo:lo + S]), "s1": _np_bits(fo.s1[lo:lo + S])}
            if fo.spec.n_states > 1:      # this rank's slice of every state after the first, back to back
                st["s2"] = np.concatenate([_np_bits(fo.s2[i * n + lo:i * n + lo + S])
                                           for i in range(fo.spec.n_states - 1)])
            out.append({"rc": int(rc), **{nm: cr.sha(v.view(np.uint8)) for nm, v in st.items()}})
        return out

    def finish(self):
        with open(os.path.join(self.out, f"rank{self.rank}.json"), "w") as f:
            json.dump(self.rec, f)


def main():
    out_dir = sys.argv[1]
    dist.init_process_group("gloo")
    os.makedirs(out_dir, exist_ok=True)
    w = Worker(out_dir)
    w.refusals()
    w.allreduce()
    w.broadcast_gather()
    w.list_api()
    w.fused_steps()
    w.finish()
    torch.cuda.synchronize()
    dist.barrier()
    w.comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
