"""Per-launch breakdown of one flagship grid step (BASELINE config 2, the step bench.py times).

torch.profiler with CUDA activities records every kernel and memset of K steps after a warm-up; each step is the
L2 flush that bench.py runs followed by one wva_grid_solve_device.  Prints, per launch, the median device time
over the steps and the median time it adds to the step (its end minus the previous launch's end: with programmatic
dependent launch a kernel starts while its predecessor drains, and its device time includes that wait), then the
median step span (first launch start to last launch end) and the idle time inside it (no launch running).
With --cells, also the median wall time of engine.grid_solve(..., want_cells=True) (cell table copied back).
With --nan, every server gets an infinite current cost on accelerator 0, which makes the value of its other
accelerators NaN and turns pruning off: every non-shared cell of a loaded row is a candidate (the worst case of
grid_sort_cands).  Also prints the candidates and chunks grid_order listed.

    python tools/grid_profile.py [--steps 50] [--trace DIR] [--cells] [--nan]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, ".")
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from workload_variant_autoscaler_b200 import Engine, _abi, config2_grid, synth_fleet  # noqa: E402


def card() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def short(name: str) -> str:
    if name.startswith("Memset") or name.startswith("Memcpy"):
        return name
    return name.split("(")[0].split("<")[0].replace("void ", "").replace("wva::", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--trace", default=None, help="also write the chrome trace into this directory")
    ap.add_argument("--cells", action="store_true", help="also time grid_solve(want_cells=True)")
    ap.add_argument("--nan", action="store_true", help="NaN values on every server: nothing pruned")
    args = ap.parse_args()

    eng = Engine(0)
    fleet, grid = synth_fleet(100, 4, seed=42), config2_grid()
    if args.nan:
        fleet.srv_cur_acc[:] = 0
        fleet.srv_cur_replicas[:] = 2
        fleet.srv_cur_cost[:] = float("inf")
    S = fleet.n_servers
    blk = torch.zeros(10 * S, dtype=torch.int32, device="cuda")
    cols = _abi.AllocsC()
    b = blk.data_ptr()
    cols.feasible = C.cast(b, _abi.u8p)
    for k, name in enumerate(("acc", "replicas", "batch"), start=1):
        setattr(cols, name, C.cast(b + 4 * S * k, _abi.i32p))
    for k, name in enumerate(("cost", "value", "itl", "ttft", "rho", "max_rate"), start=4):
        setattr(cols, name, C.cast(b + 4 * S * k, _abi.f32p))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ext = torch.cuda.ExternalStream(eng.stream)
    eng.upload(fleet)

    def steps(k):
        with torch.cuda.stream(ext):
            for _ in range(k):
                flush.fill_(1)
                eng.grid_solve_device(grid, cols)
        torch.cuda.synchronize()

    steps(10)
    l0 = eng.launch_count
    steps(args.steps)
    launches = eng.launch_count - l0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        steps(args.steps)
    path = os.path.join(args.trace or "/tmp", "grid_profile.pt.trace.json")
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
    prof.export_chrome_trace(path)
    with open(path) as fh:
        ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    ev.sort(key=lambda e: e["ts"])
    per_step, cur = [], None
    for e in ev:
        n = short(e["name"])
        if "elementwise" in n or "fill" in n.lower():  # the L2 flush opens a step
            cur = []
            per_step.append(cur)
        elif cur is not None:
            cur.append((n, float(e["ts"]), float(e["dur"])))
    per_step = [s for s in per_step if s]
    by_name, adds = {}, {}
    for s in per_step:
        seen, added, prev_end = {}, {}, s[0][1]
        for n, t, d in s:
            seen[n] = seen.get(n, 0.0) + d
            added[n] = added.get(n, 0.0) + max(t + d - prev_end, 0.0)
            prev_end = max(prev_end, t + d)
        for n, d in seen.items():
            by_name.setdefault(n, []).append(d)
            adds.setdefault(n, []).append(added[n])
    spans = [max(t + d for _, t, d in s) - s[0][1] for s in per_step]

    def busy_of(s):  # length of the union of the launches' intervals
        tot, end = 0.0, s[0][1]
        for _, t, d in sorted(s, key=lambda x: x[1]):
            if t + d > end:
                tot += t + d - max(t, end)
                end = t + d
        return tot
    busy = [busy_of(s) for s in per_step]
    print(f"device: {card()}")
    print(f"{len(per_step)} profiled steps, {launches} library launches per {args.steps} steps")
    plan = (C.c_uint32 * 31)()
    eng._L.wva_dbg_read_plan(eng._h, plan)  # item_count[2 * 256 + 1 ..]: [15] candidates, [16] chunks (grid_order)
    print(f"grid_order: {plan[15]} candidates in {plan[16]} chunks")
    order = [n for n, _, _ in per_step[0]]
    print(f"  {'launch':<22s} {'device':>8s} {'adds':>8s}")
    for n in dict.fromkeys(order):
        print(f"  {n:<22s} {statistics.median(by_name[n]):8.1f} {statistics.median(adds[n]):8.1f} us")
    print(f"  {'step span':<22s} {statistics.median(spans):8.1f} us")
    print(f"  {'idle inside span':<22s} {statistics.median([a - b for a, b in zip(spans, busy)]):8.1f} us")
    if args.cells:
        for _ in range(3):
            eng.grid_solve(fleet, grid, want_cells=True)
        ts, dev = [], []
        for _ in range(15):
            t0 = time.perf_counter()
            eng.grid_solve(fleet, grid, want_cells=True)
            ts.append(time.perf_counter() - t0)
            dev.append(eng.last_device_ms)
        print(f"grid_solve(want_cells=True): median {1e3 * statistics.median(ts):.3f} ms per call "
              f"(min {1e3 * min(ts):.3f}), device span median {statistics.median(dev):.3f} ms, {len(ts)} calls")
        n = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                eng.grid_solve(fleet, grid, want_cells=True)
        prof.export_chrome_trace(path)
        with open(path) as fh:
            ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
        tot = {}
        for e in ev:
            tot[short(e["name"])] = tot.get(short(e["name"]), 0.0) + float(e["dur"])
        print("  per call with the cell table (mean of %d):" % n)
        for k, v in tot.items():
            print(f"  {k:<22s} {v / n:10.1f} us")
    eng.close()


if __name__ == "__main__":
    main()
