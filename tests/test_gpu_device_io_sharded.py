"""The entry points of re-solving from device memory refuse a sharded handle (nranks > 1) with ERR_UNSUPPORTED: two
processes, one GPU each, join one NCCL communicator and call every one of them.  Skipped on single-GPU machines."""
import multiprocessing as mp

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _rank(rank, uid, out):
    try:
        import cosmo_b200
        from cosmo_b200 import engine as E, model as M
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(50, 80, 0.1, seed=1)
        eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], cosmo_b200.Settings(scaling=0).to_struct(),
                       device=rank)
        eng.comm_init(2, rank, uid)
        calls = {"set_caller_stream": lambda: eng.set_caller_stream(None),
                 "update_qb_original": lambda: eng.update_qb_original(q, b),
                 "original_qb": lambda: eng.original_qb(np.empty(eng.n), None),
                 "solution": lambda: eng.solution(False, np.empty(eng.n)),
                 "rescale_iterates": eng.rescale_iterates}
        codes = {}
        for name, fn in calls.items():
            try:
                fn()
                codes[name] = 0
            except E.EngineError as e:
                codes[name] = e.code
        eng.close()
        out.put((rank, codes))
    except Exception as e:   # reported to the parent instead of a silent hang
        out.put((rank, repr(e)))


def test_new_entry_points_refuse_a_sharded_handle():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from cosmo_b200 import engine as E
    uid = E.nccl_unique_id()
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, uid, out)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = dict(out.get(timeout=600) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    for rank in range(2):
        assert results[rank] == {k: E.ERR_UNSUPPORTED for k in ("set_caller_stream", "update_qb_original", "original_qb",
                                                                "solution", "rescale_iterates")}, results[rank]
