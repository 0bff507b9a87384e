"""Kernel trace of the CG reduced-KKT hot loop (bench.py's workload C2 by default).

Builds the random sparse QP, warms up, then runs K ADMM iterations under torch.profiler with CUDA activities and writes
into OUT_DIR:
  trace.json    the Chrome trace
  summary.json  per kernel name: count, total and mean us;
                per ADMM iteration: GPU busy time, the sum of the gaps between consecutive device activities, and the
                  host-poll gaps (the idle time after each device-to-host copy: the CG loop reads its done flag back);
                per CG iteration (cg_update_u .. cg_update_xr): time in the two windowed passes against everything else.
The card's name, power limit and maximum SM clock are printed and stored with it.

  python tests/run_cg_trace.py OUT_DIR [--n 50000 --m 100000 --density 0.01 --seed 2 --iters 10 --warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                                   # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % exc


def short(name):
    """Kernel name without its argument list: `spmv_win_kernel<double, cosmo::EpiScale<double>>`."""
    i = name.find("(")
    return (name[:i] if i > 0 else name).replace("void ", "").replace("cosmo::", "").strip()


def is_windowed_pass(name):
    return "spmv_win_kernel" in name and ("EpiScale" in name or "EpiKktOp" in name)


def summarize(events):
    """events: device activities (kernels and copies) of one stream sorted by start, each {name, ts, dur, kind}.

    A kernel launched as a programmatic dependent starts before its predecessor ends and waits on the device, so its
    trace duration overlaps the predecessor's.  Every time below is exclusive: an activity counts from the later of its
    start and the previous activity's end (`xdur`), so the times of consecutive kernels add up to the elapsed time."""
    prev_end = None
    for e in events:
        end = e["ts"] + e["dur"]
        e["xdur"] = max(0.0, end - max(e["ts"], prev_end)) if prev_end is not None else e["dur"]
        e["xts"] = max(e["ts"], prev_end) if prev_end is not None else e["ts"]
        prev_end = end if prev_end is None else max(prev_end, end)
    per_kernel = {}
    for e in events:
        if e["kind"] != "kernel":
            continue
        k = per_kernel.setdefault(e["name"], {"count": 0, "total_us": 0.0, "total_trace_us": 0.0})
        k["count"] += 1
        k["total_us"] += e["xdur"]
        k["total_trace_us"] += e["dur"]
    for k in per_kernel.values():
        k["mean_us"] = k["total_us"] / k["count"]

    # ADMM iterations: each one starts with the right-hand-side pass A'(rho .* x2) (the only EpiAddVec product)
    starts = [i for i, e in enumerate(events) if e["kind"] == "kernel" and "EpiAddVec" in e["name"]]
    admm = []
    for j, i0 in enumerate(starts):
        i1 = starts[j + 1] if j + 1 < len(starts) else len(events)
        seg = events[i0:i1]
        busy = sum(e["xdur"] for e in seg)
        gaps, poll = 0.0, 0.0
        for a, b in zip(seg, seg[1:]):
            g = max(0.0, b["xts"] - (a["xts"] + a["xdur"]))
            gaps += g
            if a["kind"] == "memcpy_dtoh":
                poll += g
        span = seg[-1]["xts"] + seg[-1]["xdur"] - seg[0]["xts"]
        admm.append({"span_us": span, "busy_us": busy, "gaps_us": gaps, "host_poll_gaps_us": poll,
                     "kernels": sum(1 for e in seg if e["kind"] == "kernel"),
                     "warm_start_A_scale": sum(1 for e in seg if e["kind"] == "kernel" and "EpiScale" in e["name"]) -
                                           sum(1 for e in seg if e["kind"] == "kernel" and "cg_update_u" in e["name"])})

    # CG iterations: cg_update_u .. cg_update_xr (one graph node sequence)
    cg = []
    i = 0
    while i < len(events):
        e = events[i]
        if e["kind"] == "kernel" and "cg_update_u" in e["name"]:
            j = i + 1
            while j < len(events) and not (events[j]["kind"] == "kernel" and "cg_update_xr" in events[j]["name"]):
                j += 1
            if j == len(events):
                break
            seg = events[i:j + 1]
            span = seg[-1]["xts"] + seg[-1]["xdur"] - seg[0]["xts"]
            win = sum(x["xdur"] for x in seg if x["kind"] == "kernel" and is_windowed_pass(x["name"]))
            cg.append({"span_us": span, "windowed_us": win, "other_us": span - win, "kernels": len(seg)})
            i = j + 1
        else:
            i += 1

    def stats(rows, key):
        v = np.array([r[key] for r in rows], dtype=np.float64)
        return {"mean": float(v.mean()), "median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())} if v.size else None

    # the first ADMM iteration of the window is the one after the warm-up solve's reset: report it, average the rest
    steady = admm[1:] if len(admm) > 1 else admm
    return {
        "kernels": dict(sorted(per_kernel.items(), key=lambda kv: -kv[1]["total_us"])),
        "admm_iterations": admm,
        "admm_steady": {k: stats(steady, k) for k in ("span_us", "busy_us", "gaps_us", "host_poll_gaps_us", "kernels")},
        "cg_iterations": {"count": len(cg), "kernels_per_iteration": sorted({r["kernels"] for r in cg}),
                          **{k: stats(cg, k) for k in ("span_us", "windowed_us", "other_us")}},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--m", type=int, default=100_000)
    ap.add_argument("--density", type=float, default=0.01)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import cosmo_b200
    from cosmo_b200 import model as M

    if not torch.cuda.is_available():
        raise SystemExit("run_cg_trace.py needs a CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    gpu = card()
    print("card:", gpu)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(a.n, a.m, a.density, a.seed)
    settings = cosmo_b200.Settings(scaling=0, adaptive_rho=False, max_iter=a.warmup, eps_abs=0.0, eps_rel=0.0)
    eng = cosmo_b200.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], settings.to_struct())

    def run(iters):
        st = cosmo_b200.Settings(scaling=0, adaptive_rho=False, max_iter=iters, eps_abs=0.0, eps_rel=0.0).to_struct()
        eng.update_settings(st)
        eng.reset()
        return eng.solve()

    run(max(a.warmup, 1))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = run(a.iters)
        torch.cuda.synchronize()
    trace = os.path.join(a.out_dir, "trace.json")
    prof.export_chrome_trace(trace)

    with open(trace) as f:
        raw = json.load(f)
    events = []
    for e in raw.get("traceEvents", []):
        cat = e.get("cat", "")
        if cat == "kernel":
            kind = "kernel"
        elif cat == "gpu_memcpy":
            kind = "memcpy_dtoh" if "DtoH" in e.get("name", "") else "memcpy"
        elif cat == "gpu_memset":
            kind = "memset"
        else:
            continue
        events.append({"name": short(e["name"]), "ts": float(e["ts"]), "dur": float(e.get("dur", 0.0)), "kind": kind})
    events.sort(key=lambda e: e["ts"])
    summary = summarize(events)
    summary["card"] = gpu
    summary["workload"] = {"n": a.n, "m": a.m, "density": a.density, "seed": a.seed, "iters": a.iters,
                           "cg_iters_per_admm_iter": out.kkt_inner_iterations / max(out.iter, 1),
                           "kkt_multiplications": out.kkt_multiplications, "kernel_launches": out.kernel_launches}
    with open(os.path.join(a.out_dir, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)

    print(json.dumps({"card": gpu, "workload": summary["workload"], "admm_steady": summary["admm_steady"],
                      "cg_iterations": summary["cg_iterations"]}, indent=1))
    for name, k in list(summary["kernels"].items())[:12]:
        print("%10.1f us  %6d x %9.2f us  %s" % (k["total_us"], k["count"], k["mean_us"], name))
    eng.close()


if __name__ == "__main__":
    main()
