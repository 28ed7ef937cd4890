"""Where the time of one fused solve of the benchmark's workload goes (bench.make_problem(..., fused=True): dopri5,
LinearField, 65,536 x 128 float32, the bench's options).  A diagnostic, not a bench.  Prints ONE JSON line:

  card                 nvidia-smi name, power limit and max SM clock (a query only)
  loop_ms_per_solve    CUDA events over `--solves` warm solves with the device-side loop (what bench.py times)
  step_ms_per_solve    the same with device_loop=False (the host replays the captured attempt)
  profiled             torch.profiler (CUPTI) of `--profiled` solves per mode, per solve: summed device time of each
                       kernel group, idle time between kernels on the solver stream, the gap from the end of one attempt
                       kernel to the start of the next, and the host time from the odeint call to the launch that starts
                       the attempt loop.  Kernels inside a conditional graph node may be invisible to CUPTI, so the
                       per-attempt kernels are read from the device_loop=False run; `loop_overhead_per_attempt_us` is
                       what the device loop spends per attempt beyond the attempt kernel's own time.  When the solve runs
                       as one persistent launch (k_linear_solve), `solve_kernel_us_per_attempt` is that launch's time per
                       attempt, grid barrier and controller step included.

    python scripts/solve_breakdown.py [--solves 20] [--profiled 5] [--trace-dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch                                             # noqa: E402
from torch.profiler import ProfilerActivity, profile, record_function   # noqa: E402
import bench                                             # noqa: E402
import torchdiffeq_b200 as tdq                           # noqa: E402

GROUPS = [("attempt", "k_linear_attempt"), ("solve", "k_linear_solve"), ("controller", "k_controller"),
          ("fit", "k_fit_eval")]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                               # a diagnostic: report what is missing, keep measuring
        return {"error": str(e)}


def group_of(name):
    for g, key in GROUPS:
        if key in name:
            return g
    return "startup_and_other"


def breakdown(trace_path, n_solves):
    """Per-solve figures from a chrome trace holding `n_solves` solves, each inside a `solve` user annotation that ends
    after a device synchronise (so the kernels of solve i fall inside its window on the common timeline)."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    wins = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("ph") == "X" and e.get("name") == "solve"
                  and e.get("cat") in ("user_annotation", "cpu_op"))
    kern = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") == "kernel"), key=lambda e: e["ts"])
    rt = {e["args"]["correlation"]: e for e in ev if e.get("ph") == "X" and e.get("cat") == "cuda_runtime"
          and "correlation" in e.get("args", {})}
    per = []
    for w0, w1 in wins[-n_solves:]:
        ks = [k for k in kern if w0 <= k["ts"] <= w1]
        loop_ks = [k for k in ks if group_of(k["name"]) in ("attempt", "solve")]
        if not ks:
            per.append({"kernels_visible": 0})
            continue
        stream = loop_ks[0]["args"].get("stream") if loop_ks else ks[-1]["args"].get("stream")
        ss = [k for k in ks if k["args"].get("stream") == stream]
        r = {"kernels_visible": len(ks), "kernels_on_solver_stream": len(ss)}
        for g, _ in GROUPS + [("startup_and_other", None)]:
            sel = [k for k in ss if group_of(k["name"]) == g]
            r[g + "_ms"] = sum(k["dur"] for k in sel) / 1e3
            r[g + "_launches"] = len(sel)
        idle, end = 0.0, None
        for k in ss:
            if end is not None and k["ts"] > end:
                idle += k["ts"] - end
            end = max(end or 0.0, k["ts"] + k["dur"])
        r["solver_stream_span_ms"] = (end - ss[0]["ts"]) / 1e3
        r["solver_stream_idle_ms"] = idle / 1e3
        att = [k for k in ss if group_of(k["name"]) == "attempt"]
        if att:
            gaps = [b["ts"] - (a["ts"] + a["dur"]) for a, b in zip(att, att[1:])]
            gaps.sort()
            r["attempt_kernel_us_mean"] = sum(k["dur"] for k in att) / len(att)
            r["attempt_to_attempt_gap_us_mean"] = sum(gaps) / len(gaps) if gaps else None
            r["attempt_to_attempt_gap_us_median"] = gaps[len(gaps) // 2] if gaps else None
            r["attempt_to_attempt_gap_ms_per_solve"] = sum(gaps) / 1e3
        if loop_ks:
            r["startup_device_span_ms"] = (loop_ks[0]["ts"] - ss[0]["ts"]) / 1e3
            launch = rt.get(loop_ks[0]["args"].get("correlation"))
        else:
            launch = None
        if launch is None:                               # loop body invisible: the last graph launch of the window
            gl = [e for e in rt.values() if w0 <= e["ts"] <= w1 and e["name"].startswith("cudaGraphLaunch")]
            launch = max(gl, key=lambda e: e["ts"]) if gl else None
        if launch is not None:
            r["host_call_to_loop_launch_ms"] = (launch["ts"] - w0) / 1e3
            r["loop_launch_call"] = launch["name"]
        per.append(r)
    out = {}
    for key in per[0]:
        vals = [p[key] for p in per if isinstance(p.get(key), (int, float))]
        if vals:
            out[key] = sum(vals) / len(vals)
        elif isinstance(per[0][key], str):
            out[key] = per[0][key]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=20)
    ap.add_argument("--profiled", type=int, default=5)
    ap.add_argument("--trace-dir", default=None, help="keep the chrome traces here (default: a temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "solve_breakdown.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    f, y0_host, t, _ = bench.make_problem(dev, bench.B_PER_GPU, fused=True)
    y0, t_dev = y0_host.to(dev), t.to(dev)
    res = {"card": card(), "workload": "bench.make_problem(fused=True): dopri5 LinearField 65536 x 128 f32"}

    def solve(loop, st=None):
        opts = {"graph": True, "run_ahead": 2, "device_loop": loop}
        with torch.no_grad():
            return tdq.odeint(f, y0, t_dev, method="dopri5", rtol=bench.RTOL, atol=bench.ATOL, options=opts, _stats=st)

    def timed(loop):
        st = {}
        for _ in range(3):
            solve(loop, st)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.solves):
            solve(loop)
        b.record()
        b.synchronize()
        st = {}
        solve(loop, st)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.solves, st

    ms_loop, st_loop = timed(True)
    ms_step, st_step = timed(False)
    res["solves_timed"] = args.solves
    res["loop_ms_per_solve"] = ms_loop
    res["step_ms_per_solve"] = ms_step
    res["loop_stats"] = {k: st_loop.get(k) for k in ("attempts", "nfe", "launches", "n_accept", "n_reject")}
    res["step_stats"] = {k: st_step.get(k) for k in ("attempts", "nfe", "launches", "n_accept", "n_reject")}

    tdir = args.trace_dir or tempfile.mkdtemp(prefix="tdq_breakdown_")
    os.makedirs(tdir, exist_ok=True)
    prof = {}
    for name, loop in (("device_loop_false", False), ("device_loop", True)):
        for _ in range(2):
            solve(loop)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as pr:
            for _ in range(args.profiled):
                with record_function("solve"):
                    solve(loop)
                    torch.cuda.synchronize()
        path = os.path.join(tdir, "breakdown_%s.json" % name)
        pr.export_chrome_trace(path)
        prof[name] = breakdown(path, args.profiled)
    res["profiled"] = prof
    res["profiled_solves_per_mode"] = args.profiled
    p = prof.get("device_loop_false", {})
    att = res["loop_stats"].get("attempts")
    if att and "attempt_kernel_us_mean" in p and "startup_device_span_ms" in p and not prof["device_loop"].get("solve_launches"):
        # device-loop time that is neither start-up nor attempt-kernel time, per attempt
        rest = ms_loop - p["startup_device_span_ms"] - att * p["attempt_kernel_us_mean"] / 1e3
        res["loop_overhead_ms_per_solve"] = rest
        res["loop_overhead_per_attempt_us"] = 1e3 * rest / att
    q = prof.get("device_loop", {})
    if att and q.get("solve_launches"):
        # one persistent launch ran every attempt: its time per attempt, barrier and controller step included
        res["solve_kernel_us_per_attempt"] = 1e3 * q["solve_ms"] / att
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
