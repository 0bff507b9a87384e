"""Where does engine creation (the device part of setup!) spend its time on config C2?  COSMO_B200_SETUP_DEBUG=1."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["COSMO_B200_SETUP_DEBUG"] = "1"
import numpy as np
import cosmo_b200
from cosmo_b200 import sharding
t0 = time.perf_counter()
P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(50000, 100000, 0.01, 2)
print("problem gen %.3f s" % (time.perf_counter() - t0))
for scaling in (0, 10):
    st = cosmo_b200.Settings(scaling=scaling, adaptive_rho=False, max_iter=5, eps_abs=0.0, eps_rel=0.0)
    t0 = time.perf_counter()
    shard = sharding.make_shard(P, q, A, b, sets, 0, 1)
    t1 = time.perf_counter()
    from cosmo_b200 import engine as E
    eng = E.Engine(shard.P, shard.q, shard.A, shard.b, [cosmo_b200.model.set_tuple(S) for S in shard.sets], st.to_struct(),
                   equilibrate=(scaling != 0))
    t2 = time.perf_counter()
    print("scaling=%d make_shard %.3f s, Engine() %.3f s" % (scaling, t1 - t0, t2 - t1), flush=True)
    eng.close()
