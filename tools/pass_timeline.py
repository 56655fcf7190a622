"""Timeline of bench.py's resident passes: two contexts on two streams hold the bench batch (64 x 4 MiB, 1 KB payloads by default) and
launch one pass each in turn, exactly as bench.py's `value` does; about 30 passes run under torch.profiler (CUDA activities only).
Writes every kernel's start, end, stream, grid and block as JSON under --out, and prints per step
  - the step time: from the end of one k_fused to the end of the next (a step is one pass; the two streams take turns),
  - the exposed time: the part of the step in which no k_fused runs on the device,
  - the kernels that run in those gaps,
then per k_fused its duration and how much of it each kind of kernel of the other stream overlapped (the search, the walk,
k_resolve / k_pack_slow, anything else, the other k_fused, nothing), and every other kernel's mean duration beside another stream's
k_fused and away from it, and the card's name, power limit and SM clock, read in the same run.  A run of its own: tracing slows the host, so its step times are
not bench.py's.
python tools/pass_timeline.py [--steps 30] [--warmup 5] [--payload 1024] [--out DIR (default: a new temporary directory)]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short(name):
    m = re.search(r"\b(k_\w+(?:<[^<>]*>)?)\s*\(", name)
    if m:
        return m.group(1)
    return "memset" if "emset" in name else name[:40]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q or "unknown"
    except OSError:
        return "unknown"


def union(intervals):
    out = []
    for a, b in sorted(intervals):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--payload", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import brpc_b200

    args.out = args.out or tempfile.mkdtemp(prefix="pass_timeline-")
    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    buf, data, runs, n_full, nbytes = bench.build_batch(4, 0, payload=args.payload)
    mk = lambda: brpc_b200.Context(device=0, max_batch_bytes=nbytes + (1 << 20), max_msgs=n_full + 4096, max_runs=bench.N_SOCKETS,
                                   max_resp_bytes=2 * nbytes + 96 * n_full + (8 << 20))
    ctx = mk()
    rs, msgs, resp, info = ctx.process_batch_ptr(buf.ptr, nbytes, runs)           # (bench.py's correctness gate: it tells ctx the frame size)
    assert len(msgs) == n_full and (msgs["status"] == 0).all()
    ctxs = [ctx, mk()]
    for cx in ctxs:
        cx.upload_ptr(buf.ptr, nbytes, runs)
    for s in range(args.warmup * 2):
        ctxs[s % 2].launch()
    for cx in ctxs:
        cx.wait()
    plans = [cx.resident_plan() for cx in ctxs]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(args.steps):
            ctxs[s % 2].launch()
        for cx in ctxs:
            cx.wait()
        torch.cuda.synchronize()
    trace = os.path.join(args.out, "pass.pt.trace.json")
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    ks = []
    for e in ev:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        a = e.get("args", {})
        ks.append({"name": short(e["name"]), "start_us": float(e["ts"]), "end_us": float(e["ts"]) + float(e["dur"]), "stream": a.get("stream"),
                   "grid": a.get("grid"), "block": a.get("block"), "regs": a.get("registers per thread"), "smem": a.get("shared memory")})
    ks.sort(key=lambda k: k["start_us"])
    t0 = ks[0]["start_us"] if ks else 0.0
    for k in ks:
        k["start_us"] -= t0; k["end_us"] -= t0
    fused = [k for k in ks if k["name"] == "k_fused"]
    busy = union([[k["start_us"], k["end_us"]] for k in fused])
    ends = sorted(k["end_us"] for k in fused)
    steps = []
    for i in range(1, len(ends)):
        a, b = ends[i - 1], ends[i]
        gaps, cur = [], a                          # the parts of [a, b] no k_fused covers
        for x, y in busy:
            if y <= a or x >= b:
                continue
            if x > cur:
                gaps.append((cur, x))
            cur = max(cur, y)
        if cur < b:
            gaps.append((cur, b))
        inside = sorted({k["name"] + "@s%s" % k["stream"] for k in ks if k["name"] != "k_fused" and any(k["start_us"] < g1 and k["end_us"] > g0 for g0, g1 in gaps)})
        steps.append({"step": i, "step_us": b - a, "exposed_us": sum(g1 - g0 for g0, g1 in gaps), "gap_kernels": inside})
    info = {"card": card(), "payload": args.payload, "n_msgs": int(n_full), "kernels": ks, "steps": steps, "plan": plans,
            "fused_shapes": sorted({(str(k["stream"]), str(k["block"])) for k in fused}), "fused_beside": fused_beside(ks, fused)}
    json.dump(info, open(os.path.join(args.out, "timeline.json"), "w"), indent=1)
    print("trace and timeline in", args.out)
    print("card (name, power limit, SM clock, max SM clock):", info["card"])
    for cx_i, p in enumerate(plans):
        print("plan ctx%d:" % cx_i, "; ".join("%s %d regs x %d thr, %d B smem, fits %d" % (k["name"], k["regs"], k["threads"], k["smem_bytes"], k["fits"]) for k in p))
    print("k_fused shapes (stream, block):", info["fused_shapes"])
    for s in steps:
        print("step %2d  %7.1f us  exposed %6.1f us  gaps: %s" % (s["step"], s["step_us"], s["exposed_us"], ", ".join(s["gap_kernels"])))
    if steps:
        body = steps[2:] if len(steps) > 6 else steps          # (the streams take turns, so steps alternate: means, not medians)
        st = statistics.mean(s["step_us"] for s in body); ex = statistics.mean(s["exposed_us"] for s in body)
        fz = statistics.mean(k["end_us"] - k["start_us"] for k in fused)
        print("mean step %.1f us, mean exposed %.1f us (%.0f %%), mean k_fused %.1f us" % (st, ex, 100.0 * ex / st, fz))
    beside = info["fused_beside"]
    print("k_fused and what the other stream runs beside it (us; a stretch where two of them run counts for the first named):")
    for b in beside:
        print("  k_fused %6.1f us @s%s  " % (b["dur_us"], b["stream"]) + "  ".join("%s %5.1f" % (c, b[c]) for c in CATS + ("nothing",)))
    body = beside[2:-2] if len(beside) > 8 else beside         # (the first and last passes have no other stream beside them)
    if body:
        print("mean over %d k_fused: %.1f us; " % (len(body), statistics.mean(b["dur_us"] for b in body))
              + ", ".join("%s %.1f" % (c, statistics.mean(b[c] for b in body)) for c in CATS + ("nothing",)))
    for name in sorted({k["name"] for k in ks if k["name"] != "k_fused"}):
        with_f, alone = [], []
        for k in ks:
            if k["name"] != name:
                continue
            d = k["end_us"] - k["start_us"]
            ov = sum(max(0.0, min(k["end_us"], f["end_us"]) - max(k["start_us"], f["start_us"])) for f in fused if f["stream"] != k["stream"])
            (with_f if d > 0 and ov >= 0.5 * d else alone).append(d)
        print("  %-22s mean %6.1f us beside another stream's k_fused (%d), %6.1f us otherwise (%d)"
              % (name, statistics.mean(with_f) if with_f else float("nan"), len(with_f), statistics.mean(alone) if alone else float("nan"), len(alone)))


CATS = ("k_tile_search", "k_tile_walk", "k_resolve/k_pack_slow", "other", "k_fused")


def category(name):
    if name in ("k_tile_search", "k_tile_walk", "k_fused"):
        return name
    return CATS[2] if name == "k_resolve" or name.startswith("k_pack_slow") else CATS[3]


def fused_beside(ks, fused):
    """For every k_fused: its duration and how much of it each kind of kernel of the other stream(s) overlapped."""
    out = []
    for f in fused:
        a, b = f["start_us"], f["end_us"]
        others = [(max(a, k["start_us"]), min(b, k["end_us"]), category(k["name"])) for k in ks
                  if k["stream"] != f["stream"] and k["start_us"] < b and k["end_us"] > a]
        cuts = sorted({a, b} | {x for o in others for x in o[:2]})
        row = {"stream": f["stream"], "start_us": a, "dur_us": b - a, "nothing": 0.0}
        row.update({c: 0.0 for c in CATS})
        for x, y in zip(cuts, cuts[1:]):
            on = {o[2] for o in others if o[0] < y and o[1] > x}
            row[next((c for c in CATS if c in on), "nothing")] += y - x
        out.append(row)
    return out


if __name__ == "__main__":
    main()
