#!/usr/bin/env python
"""Per-kernel GPU time of the bench.py workload (BenchCircuit<2^16>, same commit key, same blinders recipe), from a
torch.profiler capture of the CUDA kernels.

  python tools/kernel_breakdown.py [--inflight 12] [--steps 2] [--single 3] [--json OUT.json]

Two runs: `--steps` steps of `--inflight` proofs issued concurrently (one host thread + CUDA stream each, as in
bench.py's timed region), then `--single` proofs issued one at a time.  For each kernel name it prints the launches
per proof, the summed kernel time per proof and the mean time per launch, and for each run the wall time per proof.
With several proofs in flight kernels of different streams overlap, so the per-kernel sums add up to more than the
wall time: they say where the GPU's time goes, not how long a proof waits."""
import argparse
import ctypes
import json
import os
import re
import sys
import tempfile
import time
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload, commit key and blinders exactly as the benchmark makes them)


def short_name(name: str) -> str:
    """'void pb::k_msm_accumulate<128, 2>(uint4 const*, ...)' -> 'k_msm_accumulate<128, 2>'"""
    name = re.sub(r"^void ", "", name)
    depth, out = 0, []
    for ch in name:  # drop the parameter list: the first '(' at template depth 0
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            break
        out.append(ch)
    return re.sub(r"^(\w+::)+", "", "".join(out)).strip()


def profile(run, proofs):
    """Runs run() under torch.profiler; returns ({kernel: [launches, total_ms]}, wall ms per proof)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.time()
        run()
        torch.cuda.synchronize()
        wall_ms = (time.time() - t0) * 1e3
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    per = defaultdict(lambda: [0, 0.0])
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") == "kernel" and "dur" in ev:
            k = per[short_name(ev["name"])]
            k[0] += 1
            k[1] += ev["dur"] * 1e-3
    return per, wall_ms / proofs


def table(title, per, wall_ms_per_proof, proofs):
    rows = sorted(per.items(), key=lambda kv: -kv[1][1])
    total = sum(v[1] for v in per.values()) / proofs
    lines = [f"## {title}", "",
             f"wall {wall_ms_per_proof:.3f} ms per proof; kernel time {total:.3f} ms per proof", "",
             "| kernel | launches / proof | ms / proof | mean ms / launch | share |", "|---|---:|---:|---:|---:|"]
    for name, (n, ms) in rows:
        lines.append(f"| `{name}` | {n / proofs:.1f} | {ms / proofs:.4f} | {ms / n:.4f} | {100 * ms / proofs / total:.1f} % |")
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inflight", type=int, default=12)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--single", type=int, default=3, help="proofs issued one at a time")
    ap.add_argument("--json", default=None, help="also write both breakdowns to this file")
    args = ap.parse_args()

    import torch
    from plonk_b200 import Prover
    from plonk_b200._lib import check, lib

    torch.cuda.set_device(0)
    L = lib()
    check(L.pb200_init(0))
    arrays, _ = bench.build_workload("bench")
    srs_raw = ctypes.create_string_buffer(bench.SRS_POINTS * 96)
    check(L.pb200_srs_setup_from_secret(bench.mont(bench.SRS_X), bench.mont(bench.SRS_G), bench.SRS_POINTS, srs_raw))
    prover = Prover(bench.LABEL, arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, srs_raw.raw)
    wit = torch.frombuffer(bytearray(arrays.witnesses), dtype=torch.uint8)
    dev_wit = [wit.cuda() for _ in range(args.inflight)]
    proofs = [ctypes.create_string_buffer(1008) for _ in range(args.inflight)]
    pool = ThreadPoolExecutor(args.inflight)

    def one(slot, step):
        check(L.pb200_prove_dev(prover._h, dev_wit[slot].data_ptr(), arrays.n_witnesses, arrays.pi_idx, arrays.pi_vals, arrays.n_pi,
                                bench.blinders_for(step * args.inflight + slot), proofs[slot], None))

    def inflight_steps(k, base):
        def worker(slot):
            for s in range(k):
                one(slot, base + s)

        list(pool.map(worker, range(args.inflight)))

    def single(k, base):
        for s in range(k):
            one(0, base + s)

    inflight_steps(args.warmup, 0)
    single(1, 100)
    n_in = args.steps * args.inflight
    per_in, wall_in = profile(lambda: inflight_steps(args.steps, 1000), n_in)
    per_1, wall_1 = profile(lambda: single(args.single, 5000), args.single)
    gpu = torch.cuda.get_device_name(0)
    print(f"# kernel breakdown, bench.py workload on {gpu}\n")
    print(table(f"{args.inflight} proofs in flight ({n_in} proofs)", per_in, wall_in, n_in) + "\n")
    print(table(f"one proof at a time ({args.single} proofs)", per_1, wall_1, args.single))
    if args.json:
        out = {"gpu": gpu,
               "inflight": {"proofs_in_flight": args.inflight, "proofs": n_in, "wall_ms_per_proof": wall_in,
                            "kernels": {k: {"launches": v[0], "ms": v[1]} for k, v in per_in.items()}},
               "single": {"proofs": args.single, "wall_ms_per_proof": wall_1,
                          "kernels": {k: {"launches": v[0], "ms": v[1]} for k, v in per_1.items()}}}
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
