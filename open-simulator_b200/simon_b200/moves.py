"""Defragmentation / rebalancing: scoring candidate pod moves on a live snapshot (BASELINE config 5, SURVEY 8e row 3).

The reference names the use case (README.md:16) and has the primitive (NodeInfo.RemovePod,
vendor/k8s.io/kubernetes/pkg/scheduler/framework/types.go:539-585) but no implementation, so the definition is ours
(include/simon_gpu.h, "candidate-move scoring"): a move (pod, target) is evaluated on the state left by the placement
pass with the pod taken off its node; code = failing filter reasons (0 = feasible), gain = node-local score
(LeastAllocated + BalancedAllocation) of the target for the pod minus that of its current node.

Moves are independent units: the list is partitioned CONTIGUOUSLY over the ranks (one process per GPU) against a
replicated read-only snapshot; every rank scores its shard (engine.moves_upload / moves_run) and the exchange is
  * one all_reduce(MAX) of the packed best key  (gain + 1000) << 32 | (0xffffffff - global move index), and
  * one all_gather of every rank's top-k (k x 8 bytes) merged by (gain descending, move index ascending)
over NCCL when the ranks are GPUs (gloo in the CPU tests).  Nothing else crosses ranks.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

GAIN_BIAS = 1000


def shard_bounds(n_moves: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous partition: rank r gets [n*r/world, n*(r+1)/world)."""
    return (n_moves * rank) // world, (n_moves * (rank + 1)) // world


def pack_key(gain: int, move: int) -> int:
    return ((gain + GAIN_BIAS) << 32) | (0xFFFFFFFF - move)


def decode_key(key: int) -> Optional[Dict[str, int]]:
    if key == 0:
        return None
    return {"gain": (key >> 32) - GAIN_BIAS, "move": 0xFFFFFFFF - (key & 0xFFFFFFFF)}


Runner = Callable[[np.ndarray, int, int], Dict]
"""runner(moves_shard [n, 2] uint32, move_base, k) -> dict(best_key, n_feasible, topk=[(global move, gain)], ...)"""


def gpu_runner(engine, scope: int = 0) -> Runner:
    """Scores a shard on one GPU through the C ABI (simon_moves_upload + simon_moves_run); scope: abi.MOVES_SCOPE_* bits that
    admit GPU-share classes / classes with DoNotSchedule spread constraints (simon_moves_set_scope)."""
    def run(shard: np.ndarray, move_base: int, k: int) -> Dict:
        engine.moves_set_scope(scope)
        engine.moves_upload(shard, move_base)
        return engine.moves_run(k=k, want_arrays=False)
    return run


def merge_topk(lists: List[List[Tuple[int, int]]], k: int) -> List[Tuple[int, int]]:
    allm = [x for lst in lists for x in lst]
    allm.sort(key=lambda mg: (-mg[1], mg[0]))
    return allm[:k]


def search(moves: np.ndarray, runner: Runner, k: int = 16, rank: int = 0, world: int = 1,
           all_reduce_max=None, all_gather_topk=None):
    """Score this rank's contiguous shard of `moves`, then reduce: -> (best move dict or None, global top-k list, local result).

    all_reduce_max: callable(int) -> int (torch.distributed all_reduce MAX of one int64), None for a single process.
    all_gather_topk: callable(np.ndarray [k, 2] int64) -> np.ndarray [world, k, 2], None for a single process."""
    moves = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
    lo, hi = shard_bounds(len(moves), rank, world)
    res = runner(moves[lo:hi], lo, k)
    best = int(res["best_key"])
    if all_reduce_max is not None:
        best = all_reduce_max(best)
    mine = np.full((max(k, 1), 2), -1, np.int64)
    for q, (mv, g) in enumerate(res["topk"][:k]):
        mine[q] = (mv, g)
    if all_gather_topk is not None:
        allk = all_gather_topk(mine)
        lists = [[(int(a), int(b)) for a, b in part if a >= 0] for part in allk]
    else:
        lists = [[(int(a), int(b)) for a, b in mine if a >= 0]]
    return decode_key(best), merge_topk(lists, k), res


def torch_collectives(device: str):
    """The two collectives of the move search over the default process group (NCCL on GPUs, gloo on CPU)."""
    import torch
    import torch.distributed as dist

    def all_reduce_max(v: int) -> int:
        t = torch.tensor([v], dtype=torch.int64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return int(t.item())

    def all_gather_topk(a: np.ndarray) -> np.ndarray:
        t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(device)
        out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
        dist.all_gather(out, t)
        return np.stack([o.cpu().numpy() for o in out])
    return all_reduce_max, all_gather_topk


def sample_moves(n_pods: int, n_nodes: int, n_moves: int, seed: int = 5, placement: Optional[np.ndarray] = None) -> np.ndarray:
    """Candidate moves sampled uniformly: (pod among the running ones, target node) - SURVEY 8d, C5."""
    rng = np.random.RandomState(seed)
    if placement is not None:
        running = np.nonzero(np.asarray(placement) >= 0)[0]
        pods = running[rng.randint(0, max(len(running), 1), n_moves)] if len(running) else np.zeros(n_moves, np.int64)
    else:
        pods = rng.randint(0, max(n_pods, 1), n_moves)
    targets = rng.randint(0, max(n_nodes, 1), n_moves)
    return np.stack([pods, targets], 1).astype(np.uint32)
