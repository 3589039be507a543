"""wgmma implicit-GEMM convolution kernels (ops/csrc/tfy_conv.cu) against fp32 PyTorch references.

Run on an H100: ``python tests/gpu/conv_check.py [B]`` (writes a JSON report of every check).
"""
import ctypes
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_yarn_b200.keras import fastpath  # noqa: E402,F401  (declares the kernels)
from tf_yarn_b200.ops import native  # noqa: E402

lib = native.load()
dev = torch.device("cuda:0")
bf16 = torch.bfloat16
res = {}


def stream():
    return torch.cuda.current_stream().cuda_stream


def timeit(fn, reps=20):
    """Device time per call: `reps` launches captured in one CUDA graph (no host launch cost), replayed 5x."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / (5 * reps)


def report(name, got, ref, tol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-6
    bad = err > tol * denom
    ok = not bool(bad.any())
    res[name] = {"ok": ok, "max_abs_err": err.max().item(), "ref_max": denom, "bad_frac": bad.float().mean().item()}
    print(f"[{name}] ok={ok} max_err={err.max().item():.4g} ref_max={denom:.4g} bad={bad.float().mean().item():.4f}")
    if not ok:
        idx = bad.nonzero()[:6]
        for i in idx:
            t = tuple(i.tolist())
            print("   at", t, "got", got[t].item(), "ref", ref[t].item())
    return ok


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    H = W = 26
    torch.manual_seed(0)
    a = torch.randn(B, H, W, 32, device=dev).relu().to(bf16)               # NHWC, like a ReLU output
    w = (torch.randn(64, 3, 3, 32, device=dev) * 0.06).to(bf16)             # [O][kh][kw][C]
    bias = (torch.randn(64, device=dev) * 0.1).to(bf16)
    w_nchw = w.permute(0, 3, 1, 2).float()
    a_nchw = a.permute(0, 3, 1, 2).float()

    # ---------------------------------------------------------------- fprop (+bias, relu, pool)
    pooled = torch.zeros(B, 12, 12, 64, dtype=bf16, device=dev)
    code = torch.zeros(B, 12, 12, 64, dtype=torch.uint8, device=dev)
    rc = lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(),
                                      code.data_ptr(), B, H, W, 0.0, 1234, None, stream())
    torch.cuda.synchronize()
    print("fprop rc", rc)
    z = F.conv2d(a_nchw, w_nchw)                                            # fp32 reference
    zp, zi = F.max_pool2d(z, 2, return_indices=True)
    ref = (zp + bias.float().view(1, -1, 1, 1)).relu().permute(0, 2, 3, 1)
    report("fprop_pool", pooled, ref, 0.01)
    # argmax code: position inside the window
    zi = zi.permute(0, 2, 3, 1)
    iy, ix = zi // 24, zi % 24
    pos = (iy % 2) * 2 + (ix % 2)
    agree = ((code & 3).long() == pos).float().mean().item()
    on_ref = (ref > 0)
    on_agree = (((code >> 2) & 1).bool() == on_ref).float().mean().item()
    res["fprop_code"] = {"argmax_agree": agree, "gate_agree": on_agree, "ok": agree > 0.995 and on_agree > 0.995}
    print(f"[fprop_code] argmax_agree={agree:.5f} gate_agree={on_agree:.5f}")
    # dropout statistics + determinism of the mask for a given (seed, step)
    hp = torch.zeros(16, dtype=torch.float32, device=dev)
    p2 = torch.zeros_like(pooled)
    c2 = torch.zeros_like(code)
    lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), p2.data_ptr(), c2.data_ptr(), B, H, W,
                                 0.25, 1234, hp.data_ptr(), stream())
    torch.cuda.synchronize()
    kept = ((p2 != 0) | (ref.to(bf16) == 0)).float().mean().item()
    scale_ok = report("fprop_dropout_scale", torch.where(p2 != 0, p2.float() * 0.75, ref), ref, 0.01)
    frac = 1.0 - ((p2 == 0) & (ref.to(bf16) != 0)).float().sum().item() / max(1.0, (ref.to(bf16) != 0).float().sum().item())
    res["fprop_dropout"] = {"keep_frac": frac, "ok": abs(frac - 0.75) < 0.01 and scale_ok}
    print(f"[fprop_dropout] keep_frac={frac:.4f} ({kept:.4f})")

    # ---------------------------------------------------------------- dgrad
    dz = (torch.randn(B, 24, 24, 64, device=dev) * 0.5).to(bf16)
    dx = torch.full((B, H, W, 32), 7.0, dtype=bf16, device=dev)
    rc = lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), None, dx.data_ptr(), B, H, W, stream())
    torch.cuda.synchronize()
    print("dgrad rc", rc)
    dx_ref = torch.nn.grad.conv2d_input((B, 32, H, W), w_nchw, dz.permute(0, 3, 1, 2).float()).permute(0, 2, 3, 1)
    report("dgrad", dx, dx_ref, 0.01)
    dxg = torch.zeros_like(dx)
    lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), a.data_ptr(), dxg.data_ptr(), B, H, W, stream())
    torch.cuda.synchronize()
    report("dgrad_gated", dxg, dx_ref * (a.float() > 0), 0.01)

    # ---------------------------------------------------------------- wgrad
    acc = torch.full((int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()),), float('nan'), dtype=torch.float32, device=dev)
    sync = torch.zeros(1024, dtype=torch.int32, device=dev)
    dw = torch.zeros(64, 3, 3, 32, dtype=bf16, device=dev)
    dw_ref = torch.nn.grad.conv2d_weight(a_nchw, (64, 32, 3, 3), dz.permute(0, 3, 1, 2).float()).permute(0, 2, 3, 1)
    for it in range(3):                      # repeated launches: accumulator re-zeroing and barrier reuse
        rc = lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dz.data_ptr(), acc.data_ptr(), dw.data_ptr(), sync.data_ptr(),
                                       B, H, W, stream())
        torch.cuda.synchronize()
        report(f"wgrad_{it}", dw, dw_ref, 0.01)
    sv = [int(sync[0]), int(sync[32:544:32].sum()), int(sync[64])]
    res["wgrad_sync"] = {"ok": sv == [3, 0, 0], "sync": sv}
    print("wgrad rc", rc, "sync", sv)

    # ---------------------------------------------------------------- fused un-pool variants vs the 3-kernel path
    native.declare("tfy_conv3x3_c32_dgrad_unpool", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float]
                   + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p])
    native.declare("tfy_conv3x3_c32_wgrad_unpool", [ctypes.c_void_p] * 3 + [ctypes.c_float] + [ctypes.c_void_p] * 4
                   + [ctypes.c_int] * 3 + [ctypes.c_void_p])
    dp = (torch.randn(B, 12, 12, 64, device=dev) * 0.5).to(bf16)
    scale_u = 1.0 / 0.75
    dzp = torch.zeros(B, 24, 24, 64, dtype=bf16, device=dev)
    partial_u = torch.zeros(592 * 9 * 64, dtype=torch.float32, device=dev)
    cnt_u = torch.zeros(1, dtype=torch.int32, device=dev)
    db_ref = torch.zeros(64, dtype=bf16, device=dev)
    rc = lib.tfy_pool_drop_relu_bwd(dp.data_ptr(), c2.data_ptr(), dzp.data_ptr(), ctypes.c_float(scale_u), B, 24, 24,
                                    64, partial_u.data_ptr(), db_ref.data_ptr(), cnt_u.data_ptr(), stream())
    dw_a = torch.zeros(64, 3, 3, 32, dtype=bf16, device=dev)
    dw_b = torch.zeros(64, 3, 3, 32, dtype=bf16, device=dev)
    db_b = torch.zeros(64, dtype=bf16, device=dev)
    dx_a = torch.zeros(B, H, W, 32, dtype=bf16, device=dev)
    dx_b = torch.zeros(B, H, W, 32, dtype=bf16, device=dev)
    lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dzp.data_ptr(), acc.data_ptr(), dw_a.data_ptr(), sync.data_ptr(), B, H, W,
                              stream())
    lib.tfy_conv3x3_c32_dgrad(dzp.data_ptr(), w.data_ptr(), a.data_ptr(), dx_a.data_ptr(), B, H, W, stream())
    for it in range(2):
        rc1 = lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), c2.data_ptr(), ctypes.c_float(scale_u),
                                               acc.data_ptr(), dw_b.data_ptr(), db_b.data_ptr(), sync.data_ptr(), B, H,
                                               W, stream())
        rc2 = lib.tfy_conv3x3_c32_dgrad_unpool(dp.data_ptr(), c2.data_ptr(), ctypes.c_float(scale_u), w.data_ptr(),
                                               a.data_ptr(), dx_b.data_ptr(), B, H, W, stream())
        torch.cuda.synchronize()
        print("unpool rc", rc, rc1, rc2)
        report(f"wgrad_unpool_{it}", dw_b, dw_a.float(), 0.004)
        report(f"dbias_unpool_{it}", db_b, db_ref.float(), 0.01)
        report(f"dgrad_unpool_{it}", dx_b, dx_a.float(), 0.004)

    # ---------------------------------------------------------------- first-layer wgrad + bias grad (tensor core)
    native.declare("tfy_conv3x3_c1_wgrad_tc", [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
                   + [ctypes.c_int] * 3 + [ctypes.c_void_p])
    x1 = torch.rand(B, 28, 28, 1, device=dev)
    dz1 = (torch.randn(B, 26, 26, 32, device=dev) * 0.5).to(bf16)
    acc1 = torch.zeros(160 * 320, dtype=torch.float32, device=dev)
    cnt1 = torch.zeros(1, dtype=torch.int32, device=dev)
    dw1 = torch.zeros(32, 3, 3, 1, dtype=bf16, device=dev)
    db1 = torch.zeros(32, dtype=bf16, device=dev)
    x1b = x1.to(bf16).float()
    dw1_ref = torch.nn.grad.conv2d_weight(x1b.permute(0, 3, 1, 2), (32, 1, 3, 3),
                                          dz1.permute(0, 3, 1, 2).float()).permute(0, 2, 3, 1)
    db1_ref = dz1.float().sum((0, 1, 2))
    for it, (xt, f32) in enumerate([(x1, 1), (x1.to(bf16), 0), (x1, 1)]):
        rc = lib.tfy_conv3x3_c1_wgrad_tc(xt.data_ptr(), f32, dz1.data_ptr(), acc1.data_ptr(), cnt1.data_ptr(),
                                         dw1.data_ptr(), db1.data_ptr(), B, 28, 28, stream())
        torch.cuda.synchronize()
        report(f"c1_wgrad_tc_{it}", dw1, dw1_ref, 0.01)
        report(f"c1_dbias_tc_{it}", db1, db1_ref, 0.01)
    res["c1_state"] = {"ok": int(cnt1.item()) == 0}
    print("c1 rc", rc, "cnt", int(cnt1.item()))

    # ---------------------------------------------------------------- first-layer forward (tensor core)
    native.declare("tfy_conv3x3_c1_fwd_tc", [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3
                   + [ctypes.c_int] * 3 + [ctypes.c_void_p])
    w1 = (torch.randn(32, 3, 3, 1, device=dev) * 0.3).to(bf16)
    b1 = (torch.randn(32, device=dev) * 0.2).to(bf16)
    y1 = torch.zeros(B, 26, 26, 32, dtype=bf16, device=dev)
    y1_ref = (F.conv2d(x1b.permute(0, 3, 1, 2), w1.float().permute(0, 3, 1, 2)) + b1.float().view(1, -1, 1, 1)
              ).relu().permute(0, 2, 3, 1)
    for it, (xt, f32) in enumerate([(x1, 1), (x1.to(bf16), 0)]):
        y1.zero_()
        rc = lib.tfy_conv3x3_c1_fwd_tc(xt.data_ptr(), f32, w1.data_ptr(), b1.data_ptr(), y1.data_ptr(), B, 28, 28,
                                       stream())
        torch.cuda.synchronize()
        report(f"c1_fwd_tc_{it}", y1, y1_ref, 0.01)
    print("c1 fwd rc", rc)

    # ---------------------------------------------------------------- timings (hot L2; the in-graph numbers
    # come from profiles/launches_*.csv)
    t = {}
    t["fprop_pool_tc_us"] = timeit(lambda: lib.tfy_conv3x3_c32_pool_fwd(
        a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(), code.data_ptr(), B, H, W, 0.25, 1234,
        hp.data_ptr(), stream()))
    t["dgrad_tc_us"] = timeit(lambda: lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), a.data_ptr(),
                                                                 dx.data_ptr(), B, H, W, stream()))
    t["wgrad_tc_us"] = timeit(lambda: lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dz.data_ptr(), acc.data_ptr(),
                                                                 dw.data_ptr(), sync.data_ptr(), B, H, W, stream()))
    t["c1_wgrad_tc_us"] = timeit(lambda: lib.tfy_conv3x3_c1_wgrad_tc(
        x1.data_ptr(), 1, dz1.data_ptr(), acc1.data_ptr(), cnt1.data_ptr(), dw1.data_ptr(), db1.data_ptr(), B, 28, 28,
        stream()))
    t["wgrad_unpool_us"] = timeit(lambda: lib.tfy_conv3x3_c32_wgrad_unpool(
        a.data_ptr(), dp.data_ptr(), c2.data_ptr(), ctypes.c_float(scale_u), acc.data_ptr(), dw_b.data_ptr(),
        db_b.data_ptr(), sync.data_ptr(), B, H, W, stream()))
    t["dgrad_unpool_us"] = timeit(lambda: lib.tfy_conv3x3_c32_dgrad_unpool(
        dp.data_ptr(), c2.data_ptr(), ctypes.c_float(scale_u), w.data_ptr(), a.data_ptr(), dx_b.data_ptr(), B, H, W,
        stream()))
    t["pool_bwd_us"] = timeit(lambda: lib.tfy_pool_drop_relu_bwd(
        dp.data_ptr(), c2.data_ptr(), dzp.data_ptr(), ctypes.c_float(scale_u), B, 24, 24, 64, partial_u.data_ptr(),
        db_ref.data_ptr(), cnt_u.data_ptr(), stream()))
    t["c1_fwd_tc_us"] = timeit(lambda: lib.tfy_conv3x3_c1_fwd_tc(x1.data_ptr(), 1, w1.data_ptr(), b1.data_ptr(),
                                                                 y1.data_ptr(), B, 28, 28, stream()))
    t["c1_fwd_cuda_core_us"] = timeit(lambda: lib.tfy_conv3x3_c1_fwd(x1.data_ptr(), 1, w1.data_ptr(), b1.data_ptr(),
                                                                     y1.data_ptr(), B, 28, 28, 32, stream()))
    wcl = w.permute(0, 3, 1, 2)
    acl = a.permute(0, 3, 1, 2)
    dzcl = dz.permute(0, 3, 1, 2)
    t["fprop_cudnn_us"] = timeit(lambda: F.conv2d(acl, wcl))
    t["bwd_cudnn_us"] = timeit(lambda: torch.ops.aten.convolution_backward(
        dzcl, acl, wcl, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1, [True, True, False]))
    res["timings"] = t
    # ---------------------------------------------------------------- per-CTA event timelines (SM cycles)
    native.declare("tfy_conv_set_timeline", [ctypes.c_void_p])
    tl = torch.zeros(160 * 16, dtype=torch.int64, device=dev)
    launches = {
        "fprop": lambda: lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(),
                                                      code.data_ptr(), B, H, W, 0.25, 1234, hp.data_ptr(), stream()),
        "dgrad": lambda: lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), a.data_ptr(), dx.data_ptr(), B, H, W,
                                                   stream()),
        "wgrad": lambda: lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dz.data_ptr(), acc.data_ptr(), dw.data_ptr(),
                                                   sync.data_ptr(), B, H, W, stream()),
        "c1wgrad": lambda: lib.tfy_conv3x3_c1_wgrad_tc(x1.data_ptr(), 1, dz1.data_ptr(), acc1.data_ptr(),
                                                       cnt1.data_ptr(), dw1.data_ptr(), db1.data_ptr(), B, 28, 28,
                                                       stream()),
    }
    names = {"fprop": ["t0_ns", "setup", "prod_issued0", "prod_arrive0", "mma_full0", "mma_issued0", "epi_tfull0",
                       "epi_done0", "epi_tfull_last", "epi_done_last", "end", "mma_issued_last", "prod_done"],
             "dgrad": ["t0_ns", "setup", "prod_issued0", "prod_arrive0", "mma_full0", "mma_issued0", "epi_tfull0",
                       "-", "epi_tfull_last", "-", "end", "mma_issued_last", "prod_done"],
             "wgrad": ["t0_ns", "setup", "prod_issued0", "prod_arrive0", "mma_full0", "mma_issued_all", "epi_tmem_full",
                       "partials_stored", "grid_barrier", "-", "end", "-", "prod_done"],
             "c1wgrad": ["t0_ns", "setup", "built0", "built_last", "mma_full0", "mma_issued_all", "epi_tmem_full",
                         "atomics_done", "counter_done", "-", "end"]}
    res["timeline"] = {}
    for k, fn in launches.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        tl.zero_()
        lib.tfy_conv_set_timeline(tl.data_ptr())
        fn()
        torch.cuda.synchronize()
        lib.tfy_conv_set_timeline(None)
        v = tl.view(160, 16).cpu()
        used = v[:, 0] != 0
        v = v[used]
        out = {"ctas": int(used.sum()), "start_spread_ns": int(v[:, 0].max() - v[:, 0].min())}
        for j, nm in enumerate(names[k]):
            if j == 0 or nm == "-":
                continue
            col = v[:, j].float()
            out[nm] = [int(col.median()), int(col.max())]
        res["timeline"][k] = out
        print("[timeline]", k, json.dumps(out))
    print(json.dumps(t))
    ok = all(v.get("ok", True) for v in res.values() if isinstance(v, dict))
    res["all_ok"] = ok
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/conv_check.json", "w") as f:
        json.dump(res, f, indent=1)
    print("CONV CHECK", "PASS" if ok else "FAIL")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
