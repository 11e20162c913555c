#!/usr/bin/env python
"""Where the wall time of the headline search goes outside the kernel: the host side of one SearchEngine.search call.

Builds the headline engine the way bench.py does (CartPole, 4096 games, N = 50, synthetic weights seed 0, device inputs
rotated over four buffers, a 256 MiB L2 flush before every search, game ids on the device), warms up, then times at
least --seconds of searches.  Every search is cut at host clock stamps (CLOCK_MONOTONIC on both sides: Python's
time.perf_counter_ns and the library's mz_debug_host_split):

  prelude     search() entry -> the library entry point (argument checks, output allocation, IO struct, ctypes call)
  enqueue     library entry -> the kernel launch returned (device check, event record, launch set-up, cudaLaunchKernel)
  sync wait   the launch returned -> cudaStreamSynchronize returned, less the search's device_ms (ev0 -> ev1); host
              work done between the two (a caller's, while the search runs) is hidden in it
  device      device_ms
  epilogue    the synchronisation returned -> search() returned (event elapsed time, ctypes return, device_ms read)
  trailing    the torch.cuda.synchronize() bench.py adds after the call

The parts tile the wall time by construction, so the table names where the gap between the wall time and the kernel
goes.  --profile runs a torch.profiler pass instead (a separate invocation: tracing slows the host): the CUPTI kernel
duration against device_ms gives the device-side gap between the ev0 record and the kernel (start and end), and the
host duration of cudaLaunchKernel.

    python scripts/search_host_split.py [--seconds 1.0] [--repeats 3] [--profile] [--json OUT]

Needs a GPU; prints the card's name, power limit and maximum SM clock with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PARTS = ("prelude", "enqueue", "sync_wait", "device", "epilogue", "trailing")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out else {}


def headline_engine(B=4096, N=50):
    """The engine and the inputs of bench.py's headline workload (rank 0)."""
    import torch
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    cfg = load_game_module("cartpole").MuZeroConfig()
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, device=0, num_simulations=N, seed=cfg.seed)
    eng.load_weights(synthetic_weights(spec, 0))
    dev = torch.device("cuda", 0)
    rs = numpy.random.RandomState(100)
    obs = [torch.from_numpy(rs.uniform(-0.05, 0.05, size=(B, eng.obs_elems)).astype(numpy.float32)).to(dev)
           for _ in range(4)]
    noise = [torch.from_numpy(rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=B)).to(dev)
             for _ in range(4)]
    gid = torch.arange(B, dtype=torch.int64, device=dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    search = lambda i: eng.search(obs=obs[i % 4], add_exploration_noise=True, noise=noise[i % 4], game_id=gid)
    return eng, search, flush


def split_run(seconds):
    import torch
    eng, search, flush = headline_engine()
    stamps = (C.c_int64 * 4)()
    rows = []
    i, t_start = 0, None
    while True:
        flush.fill_(i & 0xFF)
        torch.cuda.synchronize()
        t0 = time.perf_counter_ns()
        out = search(i)
        t1 = time.perf_counter_ns()
        torch.cuda.synchronize()
        t2 = time.perf_counter_ns()
        assert eng.lib.mz_debug_host_split(eng._h, stamps) == 0
        s = list(stamps)
        dev_ns = out.device_ms * 1e6
        i += 1
        if i <= 20:                                  # warm-up: module load, attributes, allocator
            continue
        rows.append((s[0] - t0, s[1] - s[0], s[2] - s[1] - dev_ns, dev_ns, t1 - s[2], t2 - t1, t2 - t0))
        t_start = t_start or t0
        if t2 - t_start >= seconds * 1e9:
            break
    eng.close()
    a = numpy.asarray(rows, numpy.float64) / 1000.0                      # us
    med = numpy.median(a, axis=0)
    return {"searches": len(rows),
            "median_us": dict(zip(PARTS + ("wall",), (round(float(v), 2) for v in med))),
            "p10_us": dict(zip(PARTS + ("wall",), (round(float(v), 2) for v in numpy.percentile(a, 10, axis=0)))),
            "p90_us": dict(zip(PARTS + ("wall",), (round(float(v), 2) for v in numpy.percentile(a, 90, axis=0))))}


def profile_run(n=50):
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng, search, flush = headline_engine()
    for i in range(20):
        search(i)
    torch.cuda.synchronize()
    dev_ms = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(n):
            flush.fill_(i & 0xFF)
            torch.cuda.synchronize()
            dev_ms.append(search(i).device_ms)
            torch.cuda.synchronize()
    eng.close()
    kern, launch = [], []
    for e in prof.events():
        if "fc_search_kernel" in e.name and e.device_type.name == "CUDA":
            kern.append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
        elif e.name == "cudaLaunchKernel" and e.device_type.name == "CPU":
            launch.append(e.cpu_time_total)
    kern = numpy.asarray(kern, numpy.float64)
    ev = 1000.0 * numpy.asarray(dev_ms)
    return {"searches": n, "kernel_us_median": float(numpy.median(kern)) if kern.size else None,
            "device_ms_us_median": float(numpy.median(ev)),
            "event_gap_us_median": float(numpy.median(ev) - numpy.median(kern)) if kern.size else None,
            "cudaLaunchKernel_host_us_median": float(numpy.median(launch)) if launch else None,
            "kernels_seen": int(kern.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("search_host_split.py needs a CUDA device")
    res = {"card": card()}
    if args.profile:
        res["profile"] = profile_run()
        print(json.dumps(res["profile"]))
    else:
        res["runs"] = [split_run(args.seconds) for _ in range(args.repeats)]
        print("| part (us per search) | " + " | ".join(f"run {k + 1}: median (p10-p90)" for k in range(args.repeats)) + " |")
        print("|---|" + "---|" * args.repeats)
        for p in PARTS + ("wall",):
            print(f"| {p} | " + " | ".join(f"{r['median_us'][p]:.1f} ({r['p10_us'][p]:.1f}-{r['p90_us'][p]:.1f})"
                                          for r in res["runs"]) + " |")
    print("card:", res["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
