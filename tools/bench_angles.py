"""One variational step, new gate angles -> the value and dR/dθ, by three routes on the same gradient plan's network,
in one process, the routes alternating per repeat, host clock around synchronised steps:

  device   Angles.set_leaves (tncb_angles_gates + tncb_plan_set_leaves) + run + vjp + tncb_angles_pullback
  host     the Gate network re-staged with the new angles (host marshal + one H2D) + run + vjp + a download of the
           gradient block + a host reduction with tncb_gate_derivative
  torch    the gates rebuilt as Matrix leaves with torch ops on the GPU + network_function(on_device=True) forward and
           one backward of Re(R): it gives Re(dR/dθ) only, the other routes the complex dR/dθ

Every fsim angle is a parameter (AngleMap.every_angle); the networks are amp16 / amp20 (16- / 20-qubit, 10-round
random-circuit amplitudes) and bench.py's network, whose angle gates are all fsim.  Per line: seconds per step (median,
min, max over the repeats) of each route, the speed-ups of the device route, and the largest difference of the host
route's gradient from the device route's (relative to its largest entry) and of the torch route's real part.
A second record type times amp16's full angle Hessian: one tncb_plan_hvp_batch over P directions + one pullback,
against P single hvp + pullback calls, and says whether the rows are equal bit for bit.
The first line holds the card's name and power limit (nvidia-smi query).

usage: python tools/bench_angles.py [--repeats 5] [--networks amp16,amp20,bench] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import amplitude_nets, card, greedy  # noqa: E402


def timed(ctx, fn):
    import torch
    ctx.synchronize()
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    ctx.synchronize()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def stats(ts):
    return {"median_s": statistics.median(ts), "min_s": min(ts), "max_s": max(ts)}


def variational_step(ctx, tn, path, repeats):
    import torch
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.autograd import _with_payloads, network_function
    from tnc_b200.gates import load_gate, load_gate_derivative
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    amap = AngleMap.every_angle(tn)
    lv = leaves(tn)
    wrt = amap.leaves()
    assert all(lv[l].tensordata.gate[0] == "fsim" for l in wrt)
    plan = NetworkPlan.for_gradients(tn, path, wrt=wrt, ctx=ctx)
    plan.stage(tn)
    ang = Angles(ctx, tn, amap, plan)
    offs = plan.grad_offsets()
    rng = np.random.default_rng(5)
    P = amap.n_params

    def device(th):
        ang.set_leaves(plan, th)
        plan.run()
        G = plan.vjp_block()
        g = ang.pullback(th, G)[0]
        G.free()
        return g

    def host(th_np):
        for i, l in enumerate(wrt):                # every_angle: leaf order, then slot order
            lv[l].set_tensor_data(TensorData.Gate("fsim", (float(th_np[2 * i]), float(th_np[2 * i + 1])), False))
        plan.stage(tn)
        plan.run()
        G = plan.vjp_block()
        flat = G.to_numpy()
        G.free()
        g = np.zeros(P, dtype=np.complex128)
        for p, (l, s, _, c) in enumerate(amap.refs):
            a = lv[l].tensordata.gate[1]
            g[p] += c * np.dot(flat[offs[l]:offs[l] + 16], load_gate_derivative("fsim", a, s).reshape(-1))
        return g

    mtn = _with_payloads(tn, {l: load_gate("fsim", lv[l].tensordata.gate[1]) for l in wrt}, [0])
    f = network_function(mtn, path, wrt, ctx=ctx, on_device=True)

    def torch_route(th):
        th = th.detach().requires_grad_()
        t, ph = th[0::2], th[1::2]
        n = t.shape[0]
        M = torch.zeros((n, 4, 4), dtype=torch.complex128, device=th.device)
        M[:, 0, 0] = 1
        M[:, 1, 1] = M[:, 2, 2] = torch.cos(t).to(torch.complex128)
        M[:, 1, 2] = M[:, 2, 1] = -1j * torch.sin(t).to(torch.complex128)
        M[:, 3, 3] = torch.exp(-1j * ph.to(torch.complex128))
        R = f(*M.reshape(n, 2, 2, 2, 2).unbind(0))
        R.real.backward()
        return th.grad

    ths = [rng.uniform(-np.pi, np.pi, P) for _ in range(repeats + 1)]
    times = {"device": [], "host": [], "torch": []}
    worst = {"host": 0.0, "torch": 0.0}
    for k, th_np in enumerate(ths):
        th = torch.tensor(th_np, device="cuda")
        td, gd = timed(ctx, lambda: device(th))
        gd = gd.to_numpy()[0]
        th_h, gh = timed(ctx, lambda: host(th_np))
        tt, gt = timed(ctx, lambda: torch_route(th))
        if k == 0:
            continue                       # warm-up
        times["device"].append(td)
        times["host"].append(th_h)
        times["torch"].append(tt)
        scale = np.abs(gd).max()
        worst["host"] = max(worst["host"], float(np.abs(gh - gd).max() / scale))
        worst["torch"] = max(worst["torch"], float(np.abs(gt.cpu().numpy() - gd.real).max() / scale))
    out = {"params": P, "gate_leaves": len(wrt), "repeats": repeats}
    for r, ts in times.items():
        out[r] = stats(ts)
    out["speedup_vs_host"] = out["host"]["median_s"] / out["device"]["median_s"]
    out["speedup_vs_torch"] = out["torch"]["median_s"] / out["device"]["median_s"]
    out["max_rel_diff_host"], out["max_rel_diff_torch_real"] = worst["host"], worst["torch"]
    return out


def hvp_pair(ctx, plan, tangents):
    from tnc_b200 import DeviceTensor
    from tnc_b200._lib import check
    g, gd = C.c_void_p(), C.c_void_p()
    check(ctx._l.tncb_plan_hvp(ctx.handle, plan.handle, tangents.handle, None, None, None, None, C.byref(g), C.byref(gd)))
    return DeviceTensor.adopt(ctx, g), DeviceTensor.adopt(ctx, gd)


def hessian(ctx, tn, path, repeats):
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200._lib import check
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.tensornetwork import NetworkPlan
    amap = AngleMap.every_angle(tn)
    plan = NetworkPlan.for_hvp(tn, path, wrt=amap.leaves(), ctx=ctx)
    plan.stage(tn)
    ang = Angles(ctx, tn, amap, plan)
    P = amap.n_params
    th = torch.tensor(amap.theta0, device="cuda")
    eye = torch.eye(P, dtype=torch.float64, device="cuda")
    ang.set_leaves(plan, th)

    def batched():
        tan = ang.tangents(th, eye)
        g, gd = C.c_void_p(), C.c_void_p()
        check(ctx._l.tncb_plan_hvp_batch(ctx.handle, plan.handle, P, 0, None, None, None, tan.handle, None, None, None, None,
                                         C.byref(g), None, C.byref(gd), None))
        tan.free()
        G, Gd = DeviceTensor.adopt(ctx, g), DeviceTensor.adopt(ctx, gd)
        H = ang.pullback(th, G, Gd, eye)[0]
        G.free()
        Gd.free()
        return H

    def loop():
        rows = []
        for k in range(P):
            tan = ang.tangents(th, eye[k])
            G, Gd = hvp_pair(ctx, plan, tan)
            rows.append(ang.pullback(th, G, Gd, eye[k])[0])
            for t in (tan, G, Gd):
                t.free()
        return rows

    tb_, tl_ = [], []
    same = True
    for k in range(repeats + 1):
        t1, H = timed(ctx, batched)
        t2, rows = timed(ctx, loop)
        Hn = H.to_numpy()
        same = same and all(np.array_equal(Hn[i], r.to_numpy()[0]) for i, r in enumerate(rows))
        if k:
            tb_.append(t1)
            tl_.append(t2)
    return {"params": P, "repeats": repeats, "hvp_batch": stats(tb_), "hvp_loop": stats(tl_),
            "speedup": statistics.median(tl_) / statistics.median(tb_), "rows_bit_equal": bool(same),
            "symmetric_rel": float(np.abs(Hn - Hn.T).max() / np.abs(Hn).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--networks", default="amp16,amp20,bench")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import tnc_b200 as tb
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)

    def emit(rec):
        lines.append(rec)
        print(json.dumps(rec), flush=True)

    ctx = tb.Context(0)
    for name in args.networks.split(","):
        if name == "bench":
            import bench
            tn = bench.build_network()
        else:
            tn = amplitude_nets(int(name[3:]), 10, int(name[3:]), 1)[0]      # (amp16 of all zeros is exactly 0)
        path = greedy(tn)
        emit({"record": "variational_step", "network": name, **variational_step(ctx, tn, path, args.repeats)})
        if name == "amp16":
            emit({"record": "angle_hessian", "network": name, **hessian(ctx, tn, path, args.repeats)})
        ctx.trim()
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
