"""Move scope timing: 1M candidate moves on a 10k-node cluster whose GPU-share pods were placed by the engine (so they hold device
memory), scored unscoped and with GPU share + hard spread in scope, alternating, on the same list; then 20,000 moves against the
scoped checker (tests/checkers.c on the CPU oracle)."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
from simon_b200 import abi, compiler as K, moves as M, simulator, synth
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--replicas", type=int, default=10)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--moves", type=int, default=1000000)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--check", type=int, default=20000, help="moves compared with the scoped checker")
a = ap.parse_args()
SCOPE = abi.MOVES_SCOPE_GPU_SHARE | abi.MOVES_SCOPE_HARD_SPREAD

t0 = time.time()
cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, replicas=a.replicas, n_apps=10, seed_no=3, gpu_pct=a.gpu_pct)
p = simulator.plan(cluster, apps)
c = K.compile_cluster(p.nodes, p.pods, p.ctx)
blob, off = c.pods["class_blob"], c.pods["class_off"]
word = lambda w: np.array([int(blob[int(off[k]) + w]) for k in range(len(off) - 1)], np.int64)
gpu_cls, n_hard = word(K.SCW_GPU_MEM) > 0, word(K.SCW_N_PTS_HARD)
print(f"cluster: {c.n_nodes} nodes ({int((c.snap['gpu_count'] > 0).sum())} with GPUs), {len(p.pods)} pods, "
      f"{int(gpu_cls.sum())} GPU-share and {int((n_hard > 0).sum())} hard-spread classes of {len(gpu_cls)}; built in {time.time() - t0:.1f} s", flush=True)

with Engine(c, device=0) as eng:
    out = eng.schedule()[0]
    print(f"placement: {int((out >= 0).sum())} placed, {int((out == -1).sum())} unschedulable, {eng.last_kernel_ms():.1f} ms", flush=True)
    mv = M.sample_moves(len(out), c.n_nodes, a.moves, seed=11, placement=out)
    eng.moves_upload(mv, 0)
    res = {0: [], SCOPE: []}
    for scope in (0, SCOPE):                                   # warm-up of both variants
        eng.moves_set_scope(scope)
        eng.moves_replay(3)
    for _ in range(a.reps):                                    # alternating, same list
        for scope in (0, SCOPE):
            eng.moves_set_scope(scope)
            res[scope].append(eng.moves_replay(a.steps) / a.steps)
    runs = {}
    for scope in (0, SCOPE):
        eng.moves_set_scope(scope)
        runs[scope] = eng.moves_run(k=16, want_arrays=True, want_gpu_slots=bool(scope & abi.MOVES_SCOPE_GPU_SHARE))

# algorithmic bytes: 280 per move (DESIGN 3.3) + per hard constraint evaluated 88 (entry row 64, minimum / bitmap-offset pair 8,
# bitmap word and counter at the target 8, at the source 8) + per GPU filter evaluated 100 (device record 96, slot output 4)
code = runs[SCOPE]["code"]
cls = c.pods["pod_class"][mv[:, 0]]
gpu_code = 1 << abi.SFC_GPU
after_fit = (code == 0) | ((code & ((3 << abi.SFC_PTS_MISSING) | (7 << abi.SFC_IPA_AFF) | gpu_code)) != 0)
reach_gpu = gpu_cls[cls] & ((code == 0) | (code == gpu_code))
alg = 280 * a.moves + 88 * int(n_hard[cls][after_fit].sum()) + 100 * int(reach_gpu.sum())
for scope, name in ((0, "unscoped"), (SCOPE, "scoped  ")):
    ms = np.array(res[scope])
    by = 280 * a.moves if scope == 0 else alg
    print(f"{name}: {ms.min() * 1e3:.1f} / {np.median(ms) * 1e3:.1f} / {ms.max() * 1e3:.1f} us per {a.moves} moves (min / median / max of {a.reps}) "
          f"-> {a.moves / np.median(ms) * 1e3 / 1e9:.2f} G moves/s; {by / a.moves:.1f} B/move -> {by / np.median(ms) * 1e3 / 1e9:.0f} GB/s algorithmic")
nm0, nm1 = int((runs[0]["code"] == abi.MOVE_NOT_MOVABLE).sum()), int((code == abi.MOVE_NOT_MOVABLE).sum())
print(f"NOT_MOVABLE: {nm0} unscoped -> {nm1} scoped ({nm0 - nm1} moves left it); feasible {runs[0]['n_feasible']} -> {runs[SCOPE]['n_feasible']}; "
      f"feasible GPU-share moves with device slots: {int((runs[SCOPE]['gpu_slots'] != 0).sum())}")
if a.check:
    import checkers
    from oracle.binding import Oracle
    t1 = time.time()
    o = Oracle(c, threads=min(32, os.cpu_count() or 1))
    ref = o.schedule()[0]
    same = bool(np.array_equal(ref, out))
    g, cd, sl = checkers.moves_score(o, mv[:a.check], out, SCOPE)
    ok = same and np.array_equal(g, runs[SCOPE]["gain"][:a.check]) and np.array_equal(cd, code[:a.check]) and \
        np.array_equal(sl, runs[SCOPE]["gpu_slots"][:a.check])
    print(f"checker on {a.check} moves: {'PASS' if ok else 'FAIL'} (placements equal: {same}; {time.time() - t1:.0f} s)")
    if not ok:
        sys.exit(1)
