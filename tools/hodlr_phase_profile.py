# -*- coding: utf-8 -*-
"""Per-kernel device time of the HODLR factorisation, up-sweep and solve of the bench workload, from torch.profiler.

    python tools/hodlr_phase_profile.py --out DIR [--root TREE] [--workload cfg3] [--n N] [--steps 3] [--warmup 2]

Runs ``--warmup`` + ``--steps`` x (``compute`` + ``dot_solve``) of ``bench.py``'s workload through the C ABI (like
``tools/profile_step.py``) and profiles the last ``--steps`` with CUDA activities, in a run of its own.  ``--root``
imports ``bench`` and ``george_b200`` from another checkout, so that two builds can be compared in one session.

The GPU timeline of each step is cut into three windows:
  * factor: from the start of the leaf factorisation (``leaf_factor*`` or ``leaf_build_factor``) to the end of the last
    ``a2_tick`` of the ACA loop that runs beside it on a second stream.  Besides the common fields below it reports
    ``leaf_ms`` (span of the leaf kernel), ``a2_init_start_ms`` (start of ``a2_init`` after the first leaf activity)
    and ``aca_busy_ms`` (union of the ``a2_*`` kernels): an ``a2_init`` that starts only near the end of ``leaf_ms``
    means the ACA waited for the leaves;
  * up-sweep: from the start of ``finalize_panels_kernel`` to the end of the last activity before ``compute``'s
    device-to-host copy of the log-determinants (panel finalisation, leaf solve, level sweeps);
  * solve: from ``dot_solve``'s device-to-device copy of the right-hand side to the end of ``dot_kernel``.
For each window DIR/summary.json gets the device time per kernel (``finalize_panels``, ``leaf_solve<COLS>``,
``gram_tn``, ``gram_tn_small<RQ>``, ``small_solve``, ``update_nn``, ``memset``, ...) and launches per step, the span
of the window, and the idle time inside it (span minus the union of the activities).  Numbers taken under the
profiler are for attribution; step times come from ``bench.py``.
"""
import argparse
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def kernel_key(name, cat):
    """Stable short name of one GPU activity of the trace."""
    if cat == "gpu_memset":
        return "memset"
    if cat == "gpu_memcpy":
        m = re.search(r"(HtoD|DtoH|DtoD|HtoH|PtoP)", name)
        return "memcpy_" + (m.group(1) if m else "other")
    n = name[5:] if name.startswith("void ") else name
    n = n.split("(", 1)[0].replace("bgp::", "").strip()
    n = re.sub(r"_kernel(?=<|$)", "", n)
    return n


def gpu_activities(trace):
    """(start_us, end_us, key) of every kernel / memset / memcpy of a chrome trace, sorted by start."""
    out = []
    for e in trace.get("traceEvents", []):
        cat = e.get("cat", "")
        if cat not in ("kernel", "gpu_memset", "gpu_memcpy") or "dur" not in e:
            continue
        ts = float(e["ts"])
        out.append((ts, ts + float(e["dur"]), kernel_key(e.get("name", ""), cat)))
    out.sort()
    return out


def is_leaf_factor(key):
    return key.startswith("leaf_factor") or key == "leaf_build_factor"


def union_ms(acts):
    """Time covered by at least one of the activities, in ms."""
    busy, cur0, cur1 = 0.0, None, None
    for a0, a1, _ in sorted(acts):
        if cur1 is None or a0 > cur1:
            if cur1 is not None:
                busy += cur1 - cur0
            cur0, cur1 = a0, a1
        else:
            cur1 = max(cur1, a1)
    if cur1 is not None:
        busy += cur1 - cur0
    return busy * 1e-3


def windows(acts):
    """Cut the sorted activities into per-step (kind, [activities]) windows, kind "factor", "upsweep" or "solve"."""
    res = []
    i, n = 0, len(acts)
    dtod = None  # the latest device-to-device copy since the last up-sweep: where a solve starts
    while i < n:
        k = acts[i][2]
        if is_leaf_factor(k):
            j = i
            while j < n and acts[j][2] != "finalize_panels":
                j += 1
            ticks = [t for t in range(i, j) if acts[t][2] == "a2_tick"]
            res.append(("factor", acts[i:ticks[-1] + 1] if ticks else acts[i:j]))
            i, dtod = j, None
            continue
        if k == "finalize_panels":
            j = i
            while j < n and acts[j][2] != "memcpy_DtoH":
                j += 1
            res.append(("upsweep", acts[i:j]))
            i, dtod = j, None
            continue
        if k == "memcpy_DtoD":
            dtod = i
        elif k == "dot" and dtod is not None:
            res.append(("solve", acts[dtod:i + 1]))
            dtod = None
        i += 1
    return res


def summarise(acts):
    """Per-window totals averaged over the steps found: span, busy (union of activities), idle, per-kernel time."""
    out = {}
    for kind, w in windows(acts):
        s = out.setdefault(kind, {"steps": 0, "span_ms": 0.0, "busy_ms": 0.0, "idle_ms": 0.0, "kernels": {}})
        s["steps"] += 1
        if not w:
            continue
        t0, t1 = w[0][0], max(a[1] for a in w)
        for a0, a1, key in w:
            kk = s["kernels"].setdefault(key, {"ms": 0.0, "launches": 0})
            kk["ms"] += (a1 - a0) * 1e-3
            kk["launches"] += 1
        busy = union_ms(w)
        s["span_ms"] += (t1 - t0) * 1e-3
        s["busy_ms"] += busy
        s["idle_ms"] += (t1 - t0) * 1e-3 - busy
        if kind == "factor":
            leaf = [a for a in w if is_leaf_factor(a[2])]
            init = [a[0] for a in w if a[2] == "a2_init"]
            s["leaf_ms"] = s.get("leaf_ms", 0.0) + (max(a[1] for a in leaf) - leaf[0][0]) * 1e-3
            s["a2_init_start_ms"] = s.get("a2_init_start_ms", 0.0) + ((init[0] - leaf[0][0]) * 1e-3 if init else 0.0)
            s["aca_busy_ms"] = s.get("aca_busy_ms", 0.0) + union_ms([a for a in w if a[2].startswith("a2_")])
    for s in out.values():
        k = max(s["steps"], 1)
        for f in ("span_ms", "busy_ms", "idle_ms", "leaf_ms", "a2_init_start_ms", "aca_busy_ms"):
            if f not in s:
                continue
            s[f] /= k
        for v in s["kernels"].values():
            v["ms"] /= k
            v["launches"] /= k
        s["kernels"] = dict(sorted(s["kernels"].items(), key=lambda kv: -kv[1]["ms"]))
    return out


def format_summary(summary, header=""):
    lines = [header] if header else []
    for kind in ("factor", "upsweep", "solve"):
        s = summary.get(kind)
        if not s and kind == "factor":  # a trace without the factorisation (older callers cut only the sweeps)
            continue
        if not s:
            lines.append("{0}: not found in the trace".format(kind))
            continue
        lines.append("{0}: span {1:.3f} ms/step = busy {2:.3f} + idle {3:.3f} (mean of {4} steps)".format(
            kind, s["span_ms"], s["busy_ms"], s["idle_ms"], s["steps"]))
        if kind == "factor":
            lines.append("  leaf kernel span {0:.3f} ms, a2_init starts at +{1:.3f} ms, ACA kernels busy {2:.3f} ms".format(
                s["leaf_ms"], s["a2_init_start_ms"], s["aca_busy_ms"]))
        for name, v in s["kernels"].items():
            lines.append("  {0:<28s} {1:8.3f} ms  {2:6.1f} launches".format(name, v["ms"], v["launches"]))
    return "\n".join(lines) + "\n"


def device_info():
    info = {}
    try:
        import torch
        info["name"] = torch.cuda.get_device_name(0)
    except Exception as exc:  # reported, not fatal: the profile itself needs the device and fails on its own
        info["name_error"] = repr(exc)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip().splitlines()[0] if q.stdout.strip() else ""
    except Exception as exc:
        info["nvidia_smi_error"] = repr(exc)
    return info


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n", 1)[0])
    ap.add_argument("--out", required=True, help="output directory (summary.json, summary.txt, the trace)")
    ap.add_argument("--root", default=os.path.dirname(HERE), help="tree to import bench and george_b200 from")
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--n", type=int, default=0, help="number of points (default: the workload's)")
    ap.add_argument("--steps", type=int, default=3, help="profiled steps")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--exhaust", default="lowrank", choices=["dense", "lowrank"])
    ap.add_argument("--label", default="")
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    root = os.path.abspath(a.root)
    sys.path.insert(0, root)
    import bench
    wl = bench.WORKLOADS[a.workload]
    n = a.n or wl["n"]
    x, yerr, y = bench.make_data(n)
    k = bench.make_kernel(a.workload)
    os.makedirs(a.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from george_b200.solvers._hodlr import HODLRSolver
    torch.cuda.init()
    s = HODLRSolver()

    def step():
        s.compute(k, x[:, None], yerr, min_size=wl["min_size"], tol=wl["tol"], seed=42, exhaust=a.exhaust)
        return s.log_determinant, s.dot_solve(y)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:  # a short first session: the tracer can miss its start
        step()
        torch.cuda.synchronize()
    outs = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            outs.append(step())
        torch.cuda.synchronize()
    trace_path = os.path.join(a.out, "hodlr_phases.pt.trace.json")
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as fh:
        acts = gpu_activities(json.load(fh))
    summary = summarise(acts)
    meta = {"label": a.label, "root": root, "workload": wl["label"], "N": n, "steps": a.steps, "device": device_info(),
            "log_determinant": outs[-1][0], "dot_solve": outs[-1][1],
            "note": "device time under torch.profiler (CUDA activities); attribution only, step times come from bench.py"}
    with open(os.path.join(a.out, "summary.json"), "w") as fh:
        json.dump(dict(meta, phases=summary), fh, indent=1)
    text = format_summary(summary, "{0} {1} N={2} on {3}".format(a.label, wl["label"], n, meta["device"]))
    with open(os.path.join(a.out, "summary.txt"), "w") as fh:
        fh.write(text)
    sys.stdout.write(text)


if __name__ == "__main__":
    main()
