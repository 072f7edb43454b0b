"""The measurement mechanics the tools/bench_*.py scripts share: the card record, graph capture, alternated timed
windows, host-sync counts, one profiled call and the JSON record.  What a tool measures stays in the tool."""
import argparse
import json
import os
import statistics
import subprocess
import time
import warnings

import torch
from torch.profiler import ProfilerActivity, profile

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def card():
    """The card's name, power limit and SM clocks, read when the numbers they go with are taken."""
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk, clk_max = (s.strip() for s in q.split(","))
        info.update(name=name, power_limit=power, sm_clock=clk, max_sm_clock=clk_max)
    except Exception as e:  # noqa: BLE001 -- a missing nvidia-smi leaves the torch name
        info["power_limit"] = f"unknown ({type(e).__name__})"
    return info


def cuda_device(tool):
    if not torch.cuda.is_available():
        raise SystemExit(f"{tool}: needs a CUDA device (there is no CPU measurement)")
    return torch.device("cuda:0")


def arg_parser(doc, iters, frames=None, rounds=5):
    """--iters (unless None), --rounds, --frames (when the tool times training frames) and --json."""
    ap = argparse.ArgumentParser(description=doc, formatter_class=argparse.RawDescriptionHelpFormatter)
    if iters is not None:
        ap.add_argument("--iters", type=int, default=iters, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=rounds, help="timed windows per arm")
    if frames is not None:
        ap.add_argument("--frames", type=int, default=frames, help="training frames per timed window")
    ap.add_argument("--json", default=None, help="also write the result record here")
    return ap


def capture(fn, warmup, reset=None):
    """`fn` run `warmup` times on a side stream, then `reset()` if given, then captured once in a CUDA graph:
    (the graph, what the captured call of `fn` returned)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    if reset is not None:
        reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


def graph_replay(fn, warmup, reset=None):
    """The replay of `capture(fn, warmup, reset)`'s graph."""
    return capture(fn, warmup, reset)[0].replay


def alternate(arms, n, rounds, warmup):
    """Seconds per call of each arm (name -> fn), one value per round.  Every arm is warmed `warmup` times, then each
    round gives every arm in turn one window of `n` calls, timed by the host clock between two device syncs."""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) / n)
    return times


def stats(values, scale=1.0, nd=None):
    r = (lambda v: v) if nd is None else (lambda v: round(v, nd))
    return {"median": r(statistics.median(values) * scale), "min": r(min(values) * scale),
            "max": r(max(values) * scale)}


def host_syncs(fn):
    """Host synchronisations of one call of `fn`, as torch's sync debug mode reports them."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(m.message).lower() for m in caught)


def kernel_events(fn):
    """One profiled call of `fn`: its CUDA kernel events (copies and memsets dropped) and
    {"device_ms": their summed device time, "launches": their count}."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name]
    return ev, {"device_ms": sum(e.device_time for e in ev) / 1e3, "launches": len(ev)}


def emit(result, path):
    """Print the record; with a path, also write it there."""
    print(json.dumps(result, indent=1))
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump(result, f, indent=1)
