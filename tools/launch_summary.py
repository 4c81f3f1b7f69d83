#!/usr/bin/env python
"""Per-kernel launch table (kernel, launches, avg / min / max us, share) from a torch.profiler run with CUDA activities.

  python tools/launch_summary.py bench [--units 8] [--features 2000] [--steps 50]
      the resident loop of bench.py (`value`): inputs resident on the device, two submissions in flight
  python tools/launch_summary.py seq [--frames 6]
      sequence mode, one push at a time, plain launches (the workload of tools/run_seq.py)

Run each workload in a process of its own.  The table also lists torch's own kernels (the bench loop's cache flush).  The
last line compares the launches of the library's kernels (names `k_*`) the profiler saw with those the library counted:
CUPTI may not report kernels launched into the SM partition's green contexts, and if the counts differ the table is
partial -- rerun with VO_OPT_SM_PARTITION=0 (the context then never partitions the SMs) and say so beside it.
`--trace FILE` keeps the Chrome trace; otherwise it goes to a temporary directory.
"""
import argparse
import collections
import json
import os
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))


def kernel_table(trace_path):
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    agg = collections.OrderedDict()
    for e in events:
        if e.get("cat") != "kernel":
            continue
        name = e["name"].split("(")[0].split("<")[0]
        if name.startswith("void "):
            name = name[5:]
        a = agg.setdefault(name, [0, 0.0, 1e30, 0.0])
        d = float(e["dur"])
        a[0] += 1; a[1] += d; a[2] = min(a[2], d); a[3] = max(a[3], d)
    return agg


def print_table(agg, library_launches):
    tot = sum(a[1] for a in agg.values())
    print(f"{'kernel':28s} {'launches':>8s} {'avg us':>10s} {'min us':>10s} {'max us':>10s} {'share':>7s}")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:28s} {a[0]:8d} {a[1]/a[0]:10.1f} {a[2]:10.1f} {a[3]:10.1f} {100*a[1]/max(tot, 1e-9):6.1f}%")
    seen = sum(a[0] for k, a in agg.items() if k.startswith("k_"))       # the library's kernels (torch's own are listed too)
    print(f"total {tot:.1f} us; the profiler saw {seen} launches of the library's kernels, the library counted {library_launches}")


def run_bench(args, torch, profile):
    import bench
    from visual_odom_b200 import synth
    from visual_odom_b200.capi import Context
    B, w, h = args.units, bench.W_IMG, bench.H_IMG
    units = [synth.stereo_unit(w, h, s, cal=synth.KITTI00) for s in range(B)]
    pinned = []
    for u in units:
        d = {}
        for k in ("l0", "r0", "l1", "r1"):
            t = torch.empty((h, w), dtype=torch.uint8, pin_memory=True)
            t.numpy()[:] = u[k]
            d[k] = t.numpy()
        d["_keep"] = None
        pinned.append(d)
    ctx = Context(0, max_features=max(2048, args.features), max_units=bench.E2E_DEPTH * B)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    if os.environ.get("VO_OPT_SM_PARTITION") is not None:
        ctx.set_option("sm_partition", float(os.environ["VO_OPT_SM_PARTITION"]))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    pt = bench.Point(ctx, torch, stream, flush, pinned, args.features, B, w, h, units[0]["P_l"], units[0]["P_r"],
                     torch.cuda.synchronize, 1)
    pt.measure_resident(args.steps, 5, 1)           # warm-up: module loads, partition, graphs
    torch.cuda.synchronize()
    l0 = ctx.kernel_launches()
    with profile:
        pt.resident_steps(args.steps)
        torch.cuda.synchronize()
    return ctx.kernel_launches() - l0


def run_seq(args, torch, profile):
    from run_seq import stereo_frames
    from visual_odom_b200.capi import Context
    frames, P_l, P_r = stereo_frames(args.frames)
    ctx = Context(0, max_features=4096, max_units=1)
    ctx.set_option("graphs", 0)
    ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    ctx.seq_push(frames[1][0], frames[1][1], want_points=False)      # warm-up push
    torch.cuda.synchronize()
    l0 = ctx.kernel_launches()
    with profile:
        for k in range(2, args.frames + 1):
            ctx.seq_push(frames[k][0], frames[k][1], want_points=False)
        torch.cuda.synchronize()
    return ctx.kernel_launches() - l0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("workload", choices=["bench", "seq"])
    ap.add_argument("--units", type=int, default=8)
    ap.add_argument("--features", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--trace", default=None, help="keep the Chrome trace here")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("launch_summary.py needs a CUDA device")
    prof = profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
    launches = (run_bench if args.workload == "bench" else run_seq)(args, torch, prof)
    with tempfile.TemporaryDirectory() as tmp:
        path = args.trace or os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        agg = kernel_table(path)
    print(f"{torch.cuda.get_device_name(0)}, workload {args.workload}, "
          f"VO_OPT_SM_PARTITION={os.environ.get('VO_OPT_SM_PARTITION', 'default')}")
    print_table(agg, launches)


if __name__ == "__main__":
    main()
