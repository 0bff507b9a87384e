"""Measurement helper (not a test): iterations to Solved and device time per iteration of each Anderson accelerator
family on one GPU, next to EmptyAccelerator, on the mid-size QP of run_aa_timing.py.  Prints the card and its power
limit, then one JSON line per run."""
import json
import subprocess
import sys

sys.path.insert(0, ".")
import cosmo_b200

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip(), flush=True)
P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(20000, 40000, 0.005, seed=2)
families = [("EmptyAccelerator", {}), ("Type2{QRDecomp}/Restarted", {}),
            ("Type2{NormalEquations}/Restarted", dict(accelerator_type="Type2{NormalEquations}")),
            ("Type2{NormalEquations}/Rolling", dict(accelerator_type="Type2{NormalEquations}", accelerator_memory="RollingMemory")),
            ("Type1/Restarted", dict(accelerator_type="Type1")),
            ("Type1/Rolling", dict(accelerator_type="Type1", accelerator_memory="RollingMemory"))]
for name, var in families:
    for max_iter in (200, 5000):   # a fixed-length run (time per iteration) and the run to the default tolerance
        acc = "EmptyAccelerator" if name == "EmptyAccelerator" else "AndersonAccelerator"
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(accelerator=acc, scaling=0, max_iter=max_iter,
                                                        eps_abs=1e-14 if max_iter == 200 else 1e-5,
                                                        eps_rel=1e-14 if max_iter == 200 else 1e-5, **var))
        res = model.optimize()
        dev = res.times["iter_time_device"]
        stats = model.engine.accelerator_stats() if acc != "EmptyAccelerator" else {}
        print(json.dumps({"family": name, "max_iter": max_iter, "status": res.status, "iter": res.iter,
                          "safeguarding_iter": res.safeguarding_iter, "ms_per_iter": round(1e3 * dev / max(res.iter, 1), 4),
                          "launches_per_iter": round(res.kernel_launches / max(res.iter, 1), 2), **stats}), flush=True)
        model.empty_model()
