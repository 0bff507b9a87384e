"""Row sharding of the ADMM hot path across GPUs (SURVEY.md 8e).

One process per GPU.  Whole cones are assigned to ranks (SOC / PSD cones are
atomic; Zero / Nonneg / Box rows are split anywhere), contiguously and in cone
order, balanced by nnz(A[row,:]) plus the eigensolver weight |c|^3 the
reference's clique-merge heuristic uses (clique_merging.jl:403).  Rank g owns
A[R_g,:] and the m-vectors restricted to R_g; n-vectors, P and q are
replicated.  The only data-path collective is one ncclAllReduce(sum) of an
n-vector per operator application (plus max/sum reductions of a few scalars at
the reference's own check points) -- issued inside libcosmo_b200.so.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import scipy.sparse as sp

from . import engine as _eng
from . import model as M


@dataclass
class Shard:
    P: sp.csc_matrix
    q: np.ndarray
    A: sp.csc_matrix          # local rows
    b: np.ndarray
    sets: list                # local cones
    rows: np.ndarray          # global row index of every local row
    rank: int
    world: int


def _row_weights(A: sp.csc_matrix, sets) -> np.ndarray:
    m = A.shape[0]
    w = np.bincount(A.indices, minlength=m).astype(np.float64) + 1.0
    off = 0
    for S in sets:
        if isinstance(S, (M.PsdCone, M.PsdConeTriangle)) and S.dim > 0:
            w[off:off + S.dim] += float(S.sqrt_dim) ** 3 / S.dim
        off += S.dim
    return w


def partition_rows(A: sp.csc_matrix, sets, world: int) -> List[List[Tuple[int, int, int]]]:
    """Return per-rank lists of (set_index, start, stop) with start/stop relative to the set."""
    w = _row_weights(A, sets)
    cum = np.concatenate([[0.0], np.cumsum(w)])
    total = cum[-1]
    bounds = [total * (g + 1) / world for g in range(world)]
    parts: List[List[Tuple[int, int, int]]] = [[] for _ in range(world)]
    g, off = 0, 0
    for k, S in enumerate(sets):
        if S.dim == 0:
            continue
        atomic = isinstance(S, M.ATOMIC_CONES)
        if atomic:
            mid = 0.5 * (cum[off] + cum[off + S.dim])
            while g < world - 1 and mid > bounds[g]:
                g += 1
            parts[g].append((k, 0, S.dim))
        else:
            start = 0
            while start < S.dim:
                if g == world - 1:
                    stop = S.dim
                else:
                    # last row whose cumulative weight stays within this rank's bound
                    stop = int(np.searchsorted(cum, bounds[g], side="right")) - 1 - off
                    stop = min(max(stop, start), S.dim)
                if stop > start:
                    parts[g].append((k, start, stop))
                    start = stop
                if start < S.dim and g < world - 1:
                    g += 1
        off += S.dim
    return parts


def make_shard(P, q, A, b, sets, rank: int, world: int) -> Shard:
    A = sp.csc_matrix(A)
    if world == 1:
        return Shard(sp.csc_matrix(P), np.asarray(q, dtype=np.float64), A, np.asarray(b, dtype=np.float64), list(sets),
                     np.arange(A.shape[0]), 0, 1)
    parts = partition_rows(A, sets, world)[rank]
    offs = np.concatenate([[0], np.cumsum([S.dim for S in sets])]).astype(np.int64)
    rows, local_sets = [], []
    for (k, start, stop) in parts:
        S = sets[k]
        rows.append(np.arange(offs[k] + start, offs[k] + stop))
        if isinstance(S, M.Box):
            local_sets.append(M.Box(S.l[start:stop], S.u[start:stop]))
        elif isinstance(S, (M.ZeroSet, M.Nonnegatives)):
            local_sets.append(type(S)(stop - start))
        else:
            local_sets.append(S)
    rows = np.concatenate(rows) if rows else np.zeros(0, dtype=np.int64)
    A_loc = A.tocsr()[rows, :].tocsc()
    return Shard(sp.csc_matrix(P), np.asarray(q, dtype=np.float64), A_loc, np.asarray(b, dtype=np.float64)[rows],
                 local_sets, rows, rank, world)


def create_engine(shard: Shard, settings: M.Settings, device: int = 0, dist=None, D=None, E=None, c: float = 1.0,
                  dtype=np.float64) -> _eng.Engine:
    """Build the per-rank engine; with world > 1 rank 0 creates the ncclUniqueId and
    `torch.distributed` (the plumbing) broadcasts its 128 bytes."""
    if shard.world > 1 and settings.to_struct().kkt_solver in (_eng.KKT_LDL, _eng.KKT_LDL_SUPERNODAL):
        raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "the direct LDL' KKT solver is single-GPU (use CG or reduced MINRES when sharded)")
    tuples = [M.set_tuple(S) for S in shard.sets]
    eng = _eng.Engine(shard.P, shard.q, shard.A, shard.b, tuples, settings.to_struct(), D=D,
                      E=None if E is None else np.asarray(E)[shard.rows], c=c, dtype=dtype, device=device)
    M.configure_accelerator(eng, settings)
    if shard.world > 1:
        if dist is None:
            raise _eng.EngineError(_eng.ERR_INVALID, "world > 1 needs an initialised torch.distributed module")
        obj = [_eng.nccl_unique_id() if shard.rank == 0 else None]
        dist.broadcast_object_list(obj, src=0)
        eng.comm_init(shard.world, shard.rank, obj[0])
        # Peer-memory PUSH exchange of the operator partials (CUDA IPC over NVLink; p2p_push_kernel) instead of one
        # NCCL allreduce per operator application.  Bit-identical results; the default from 4 ranks up is kept from the
        # earlier NVLink measurements and has not been re-measured on H100 (COSMO_B200_P2P=0 / 1 forces either).
        mode = os.environ.get("COSMO_B200_P2P", "auto")
        use_p2p = (mode == "1" or (mode not in ("0", "1") and shard.world >= 4)) and shard.world <= 8
        if use_p2p:
            # every rank must take the same path: export first, agree, then attach
            try:
                blob, ok = eng.p2p_export(), True
            except _eng.EngineError:
                blob, ok = b"", False
            blobs = [None] * shard.world
            dist.all_gather_object(blobs, (ok, blob))
            if all(o for o, _ in blobs):
                eng.p2p_attach(b"".join(bl for _, bl in blobs), shard.world)
    return eng
