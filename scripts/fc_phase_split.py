#!/usr/bin/env python
"""Where the time of the fused FC search goes: cycles per simulation of its phases, and the passes of its persistent loop.

Builds a copy of the library with -DMZ_FC_PHASES into a temporary directory (the in-tree library is not touched), runs
the headline workload (CartPole, 4096 games, N = 50, synthetic weights seed 0, the bench's seeded inputs) and reads the
kernel's counters.  Every group times its own game with clock64(): root, select, network (dynamics + heads + softmax),
expand and backup, plus the tree levels and selection rounds it walked.  The cycles are a game's latency, stalls behind
the other warps of its SM included, so the per-phase shares are shares of the launch's critical path.

Each game also records the %globaltimer at which it started and finished.  Games that started after the first game
finished ran in a second pass of the persistent loop (their slot was busy with an earlier game); the script counts them
and prints the spread of the start times and of the games' durations in the last search.

    python scripts/fc_phase_split.py [--levels 1 default] [--games 4096] [--searches 5] [--json OUT]

--levels runs each setting of the multi-level selection in turn: "1" sets MZ_FC_SELECT_LEVELS=1 (one tree level per
round), "default" leaves it unset.  Needs a GPU; prints one table per setting and the card it ran on.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ("root", "select", "network", "expand", "backup")


def build_instrumented(out_dir):
    from muzero_general_b200 import build as b
    objs, procs = [], []
    for src in b.SOURCES:
        obj = os.path.join(out_dir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [b.NVCC] + b.FLAGS + ["-DMZ_FC_PHASES", "-c", os.path.join(b.CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc {src}:\n{out}")
    lib = os.path.join(out_dir, "libmzb200_phases.so")
    subprocess.check_call([b.NVCC, "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return lib


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out else {}


def passes(spans):
    """spans: [n, 2] start / end ns of every game of one launch."""
    import numpy
    start, end = spans[:, 0].astype(numpy.int64), spans[:, 1].astype(numpy.int64)
    t0 = int(start.min())
    us = lambda a: [round(float(v) / 1000.0, 2) for v in a]
    dur = end - start
    return {"games_started_after_first_finish": int((start > end.min()).sum()),
            "start_us": dict(zip(("min", "median", "max"), us([0, numpy.median(start) - t0, start.max() - t0]))),
            "duration_us": dict(zip(("min", "median", "max"), us([dur.min(), numpy.median(dur), dur.max()]))),
            "launch_us": us([end.max() - t0])[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", nargs="+", default=["1", "default"])
    ap.add_argument("--games", type=int, default=4096)
    ap.add_argument("--searches", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import ctypes as C
    import numpy
    from muzero_general_b200 import _lib

    tmp = tempfile.mkdtemp(prefix="mz_phases_")
    _lib.LIB_PATH = build_instrumented(tmp)
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    lib = _lib.load_library()
    read = lib.mz_fc_phase_counters
    read.restype = C.c_int
    read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    counters = (C.c_ulonglong * 8)()
    read_spans = lib.mz_fc_phase_spans
    read_spans.restype = C.c_int
    read_spans.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]

    B, N = args.games, 50
    cfg = load_game_module("cartpole").MuZeroConfig()
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(100)
    obs = rs.uniform(-0.05, 0.05, size=(B, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=B)
    game_id = numpy.arange(B, dtype=numpy.int64)

    results = {"card": card(), "games": B, "num_simulations": N, "runs": []}
    for lv in args.levels:
        if lv == "default":
            os.environ.pop("MZ_FC_SELECT_LEVELS", None)
        else:
            os.environ["MZ_FC_SELECT_LEVELS"] = lv
        eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=cfg.seed)
        eng.load_weights(synthetic_weights(spec, 0))
        run = lambda: eng.search(obs=obs, add_exploration_noise=True, noise=noise, game_id=game_id)
        for _ in range(2):
            run()
        assert read(counters, 1) == 0
        ms = [run().device_ms for _ in range(args.searches)]
        spans = numpy.zeros((B, 2), numpy.uint64)
        assert read_spans(spans.ctypes.data_as(C.POINTER(C.c_ulonglong)), B) == 0
        assert read(counters, 1) == 0
        launch = eng.last_fc_launch
        eng.close()
        c = list(counters)
        sims = c[7]
        per_sim = {p: c[i] / sims for i, p in enumerate(PHASES)}
        total = sum(per_sim.values())
        r = {"select_levels": lv, "cycles_per_sim": per_sim, "total_cycles_per_sim": total,
             "share": {p: per_sim[p] / total for p in PHASES},
             "levels_per_sim": c[5] / sims, "rounds_per_sim": c[6] / sims,
             "kernel_ms_instrumented": sorted(ms)[len(ms) // 2], "launch": launch, "passes": passes(spans)}
        results["runs"].append(r)
        print(f"MZ_FC_SELECT_LEVELS={lv}: {r['levels_per_sim']:.2f} levels/sim, {r['rounds_per_sim']:.2f} rounds/sim, "
              f"kernel {r['kernel_ms_instrumented']:.3f} ms (instrumented build, median of {len(ms)}), launch {launch}")
        ps = r["passes"]
        print(f"last search: {ps['games_started_after_first_finish']} of {B} games started after the first game finished; "
              f"start times (us after the first) {ps['start_us']}; game durations (us) {ps['duration_us']}; "
              f"first start to last end {ps['launch_us']} us")
        print("| phase | cycles / simulation | share |\n|---|---|---|")
        for p in PHASES:
            print(f"| {p} | {per_sim[p]:.0f} | {100 * r['share'][p]:.1f} % |")
        print(f"| total | {total:.0f} | |")
    print("card:", results["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
