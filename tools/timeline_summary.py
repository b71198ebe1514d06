"""Summarise a torch.profiler chrome trace of a few training steps (written by ``PTD_TIMELINE=<prefix> python bench.py``).

    python tools/timeline_summary.py tl.rank0.json [--top 30]

Prints (1) the per-kernel-name device time table, (2) per-stream busy time, (3) for the LAST complete step: the span from
the first to the last kernel, the idle gaps of the busiest (compute) stream, and every cross-GPU kernel (ptd::fused_* /
metrics / broadcast) with its start offset, duration and what the compute stream was doing meanwhile.  Device timestamps
come from CUPTI, so this is a timeline, not a benchmark: compare shares and gaps.
"""
from __future__ import annotations

import argparse
import collections
import json
import re


def load(path):
    with open(path) as f:
        tr = json.load(f)
    evs = [e for e in tr.get("traceEvents", []) if e.get("ph") == "X" and e.get("cat", "").lower() in ("kernel", "gpu_memcpy", "gpu_memset")]
    out = []
    for e in evs:
        a = e.get("args", {})
        out.append({"name": e["name"], "ts": float(e["ts"]), "dur": float(e["dur"]), "stream": a.get("stream", e.get("tid")),
                    "cat": e["cat"].lower(), "grid": a.get("grid"), "block": a.get("block")})
    out.sort(key=lambda x: x["ts"])
    return out


def short(name, n=70):
    name = re.sub(r"\(.*$", "", name)
    name = re.sub(r"<.*>", "<>", name) if len(name) > n else name
    return name[:n]


def union_busy(evs):
    busy, end = 0.0, None
    start = None
    for e in sorted(evs, key=lambda x: x["ts"]):
        s, t = e["ts"], e["ts"] + e["dur"]
        if end is None or s > end:
            if end is not None:
                busy += end - start
            start, end = s, t
        else:
            end = max(end, t)
    if end is not None:
        busy += end - start
    return busy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trace")
    ap.add_argument("--top", type=int, default=30)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    evs = load(a.trace)
    if not evs:
        print("no device events in", a.trace)
        return
    t0 = evs[0]["ts"]
    span = evs[-1]["ts"] + evs[-1]["dur"] - t0
    print("# %s: %d device events, span %.3f ms (%d steps => %.3f ms/step under the profiler)" % (a.trace, len(evs), span / 1e3, a.steps, span / 1e3 / a.steps))
    by = collections.defaultdict(lambda: [0.0, 0])
    for e in evs:
        k = short(e["name"])
        by[k][0] += e["dur"]
        by[k][1] += 1
    tot = sum(v[0] for v in by.values())
    print("\n| kernel | ms / step | launches / step | share of kernel time |\n|---|---:|---:|---:|")
    for k, (d, n) in sorted(by.items(), key=lambda kv: -kv[1][0])[:a.top]:
        print("| `%s` | %.3f | %.1f | %.1f %% |" % (k, d / 1e3 / a.steps, n / a.steps, 100 * d / tot))
    print("| (sum of all kernels, streams overlapped) | %.3f | %.1f | |" % (tot / 1e3 / a.steps, len(evs) / a.steps))
    streams = collections.defaultdict(list)
    for e in evs:
        streams[e["stream"]].append(e)
    print("\n| stream | events | busy ms / step |\n|---|---:|---:|")
    main_stream, best = None, -1
    for s, es in streams.items():
        b = union_busy(es)
        print("| %s | %d | %.3f |" % (s, len(es), b / 1e3 / a.steps))
        if b > best:
            main_stream, best = s, b
    # ---- last complete step: delimited by the metric kernel (exactly one per step, right after the forward pass)
    marks = [e for e in evs if "metrics_kernel" in e["name"]]
    if len(marks) >= 2:
        lo, hi = marks[-2]["ts"], marks[-1]["ts"]
        step = [e for e in evs if lo <= e["ts"] < hi]
        comm_re = re.compile(r"allreduce|broadcast|metrics|barrier|push_kernel|reduce_to_caller|ll_|fused_sgd")
        comm = [e for e in step if comm_re.search(e["name"])]
        comp = [e for e in step if not comm_re.search(e["name"])]
        print("\nlast complete step (metric kernel to metric kernel): %.3f ms; compute kernels busy %.3f ms (union), "
              "communication / optimizer kernels %.3f ms (sum, overlapped with compute)" %
              ((hi - lo) / 1e3, union_busy(comp) / 1e3, sum(e["dur"] for e in comm) / 1e3))
        # the step runs [forward_k+1 ... ] after the marker; backward of step k ends where the last wgrad/dgrad/bn_bwd kernel ends
        bwd = [e for e in comp if re.search(r"wgrad|dgrad|bwd|backward", e["name"])]
        if bwd:
            bwd_end = max(e["ts"] + e["dur"] for e in bwd)
            after = [e for e in comm if e["ts"] + e["dur"] > bwd_end]
            tail_end = max([e["ts"] + e["dur"] for e in after] + [bwd_end])
            print("end of backward compute -> end of the last all-reduce / optimizer kernel (exposed tail): %.1f us" % (tail_end - bwd_end))
        print("\ncommunication / optimizer kernels of the step (offset from the marker ms, duration us, grid, concurrent compute kernel):")
        for e in comm:
            mid = e["ts"] + e["dur"] / 2
            over = [c for c in comp if c["ts"] <= mid <= c["ts"] + c["dur"]]
            print("  %7.3f  %8.1f  %-12s %-48s | %s" % ((e["ts"] - lo) / 1e3, e["dur"], e["grid"], short(e["name"], 48),
                                                        short(over[0]["name"], 40) if over else "(nothing: exposed)"))
        gaps, prev_end = [], lo
        for e in sorted(comp, key=lambda x: x["ts"]):
            if e["ts"] - prev_end > 8.0:
                gaps.append((e["ts"] - prev_end, (prev_end - lo) / 1e3, short(e["name"], 50)))
            prev_end = max(prev_end, e["ts"] + e["dur"])
        gaps.sort(reverse=True)
        print("\nlargest gaps between compute kernels (us, at offset ms, next kernel):")
        for g, off, nm in gaps[:8]:
            print("  %8.1f us  @ %7.3f ms  -> %s" % (g, off, nm))


if __name__ == "__main__":
    main()
