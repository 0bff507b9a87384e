"""C5 (MAXCUT dual SDP, |V| = 10 000, CliqueGraphMerge): the reverse of the decomposition on the host (chordal.reverse)
against the device (cosmo_b200_reverse_decomposition), without and with the completion of the dual.

The device wall time includes the copies of x, s and mu (50 005 000 rows each for s and mu) to host memory; the device
time is the kernels alone (CUDA events, the call's stats).  The first device call allocates the buffers and the dense
workspace and is reported apart.  Usage: python tests/run_reverse_timing.py [|V|] [repeats]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import cosmo_b200  # noqa: E402
from cosmo_b200 import chordal  # noqa: E402


def main():
    nv = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        card = "unknown"
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(decompose=True, reverse_on_device=True))
    t0 = time.perf_counter()
    res = model.optimize()
    print("setup + solve %.2f s (%s after %d iterations), n' = %d, m' = %d, m = %d, cliques %d (max %d)"
          % (time.perf_counter() - t0, res.status, res.iter, model.engine.n, model.engine.m, model.m,
             len(model._dec.clique_sizes), max(model._dec.clique_sizes)), flush=True)
    info, eng = model._dec, model.engine
    x2, s2, mu2 = model._x2, model._s2, model._mu2
    out = {"card": card, "nv": nv, "m_orig": model.m, "cliques": len(info.clique_sizes)}
    for cd in (False, True):
        key = "complete" if cd else "plain"
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            xh, sh, muh = chordal.reverse(info, x2, s2, mu2, complete_dual=cd)
            t.append(time.perf_counter() - t0)
        out["host_%s_s" % key] = float(np.median(t))
        t0 = time.perf_counter()
        xd, sd, mud, st = eng.reverse_decomposition(complete_dual=cd)
        out["device_first_%s_s" % key] = time.perf_counter() - t0
        td, tk = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            xd, sd, mud, st = eng.reverse_decomposition(complete_dual=cd)
            td.append(time.perf_counter() - t0)
            tk.append(st["device_us"] * 1e-3)
        out["device_wall_%s_s" % key] = float(np.median(td))
        out["device_kernels_%s_ms" % key] = float(np.median(tk))
        out["pinv_fallbacks_%s" % key] = st["pinv_fallbacks"]
        out["workspace_bytes"] = st["workspace_bytes"]
        out["same_x_s_%s" % key] = bool(np.array_equal(xd, xh) and np.array_equal(sd, sh))
        out["nonfinite_mu_host_device_%s" % key] = [int((~np.isfinite(muh)).sum()), int((~np.isfinite(mud)).sum())]
        ok = np.isfinite(muh) & np.isfinite(mud)
        out["mu_rel_maxdiff_%s" % key] = float(np.abs(mud[ok] - muh[ok]).max() / max(np.abs(muh[ok]).max(), 1e-300))
        print(json.dumps({k: v for k, v in out.items() if key in k}), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
