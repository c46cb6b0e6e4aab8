"""Times the debugger check (pb200_circuit_unsatisfied, pb200_prover_unsatisfied) against a proof (pb200_prove) for the
reference's BenchCircuit<2^16> and <2^20>, with the card's name and power limit read in the same run.  Prints one JSON
object; --out also writes it to a file outside the tree.

Per size, after one warm-up call of each: rounds of circuit-level and prover-level checks on the honest witness and on
one with a corrupted witness, and a proof on the honest witness, alternated in one process.  Each time is the wall
time of the whole call (uploads, kernels, the copies back), which synchronises before it returns.  A separate
torch.profiler run then sums the GPU time of the check's three kernels per call.

    python tools/unsatisfied_bench.py --rounds 5 --out /tmp/unsatisfied_bench.json
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import random
import re
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.compress_bench import gpu_info  # noqa: E402

R_MOD = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001


def _mont(v: int) -> bytes:
    return (v * (1 << 256) % R_MOD).to_bytes(32, "little")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-sizes", default="16,20")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import plonk_b200
    from plonk_b200 import gadgets
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    result = {"gpu": gpu_info(), "sizes": {}}
    rng = random.Random(1)
    for log_n in (int(x) for x in args.log_sizes.split(",")):
        a = gadgets.bench_circuit(1 << log_n).arrays()
        n_srs = (1 << (a.constraints + 6 - 1).bit_length()) + 7
        srs = ctypes.create_string_buffer(96 * n_srs)
        check(lib().pb200_srs_setup_from_secret(_mont(0xABCDEF), _mont(0x13579), n_srs, srs))
        prover = plonk_b200.Prover(b"debugger-bench", a.constraints, a.selectors, a.wires, a.n_witnesses, srs.raw)
        # corrupt the witness on the last constraint's output wire
        w = int.from_bytes(a.wires[4 * (3 * a.constraints - 1) : 4 * 3 * a.constraints], "little")
        bad = type(a)(a.constraints, a.selectors, a.wires, a.witnesses[: 32 * w] + _mont(rng.randrange(R_MOD)) + a.witnesses[32 * w + 32 :],
                      a.pi_idx, a.pi_vals)
        blinders = b"".join(_mont(rng.randrange(R_MOD)) for _ in range(14))
        calls = {
            "circuit_honest_ms": lambda: plonk_b200.unsatisfied_constraints(a),
            "prover_honest_ms": lambda: prover.unsatisfied_constraints(a.witnesses, a.pi_idx, a.pi_vals),
            "circuit_corrupted_ms": lambda: plonk_b200.unsatisfied_constraints(bad),
            "prover_corrupted_ms": lambda: prover.unsatisfied_constraints(bad.witnesses, bad.pi_idx, bad.pi_vals),
            "prove_ms": lambda: prover.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders),
        }
        failing = len(calls["circuit_corrupted_ms"]())
        for f in calls.values():
            f()
        times = {k: [] for k in calls}
        for _ in range(args.rounds):
            for k, f in calls.items():
                t0 = time.perf_counter()
                f()
                times[k].append((time.perf_counter() - t0) * 1e3)
        size = {k: round(statistics.median(v), 3) for k, v in times.items()}
        size["failing_rows_corrupted"] = failing
        size["constraints"] = a.constraints

        import torch
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                calls["prover_corrupted_ms"]()
            torch.cuda.synchronize()
        us, all_us = {}, 0.0
        for e in prof.events():
            if e.device_type != DeviceType.CUDA:
                continue
            all_us += e.time_range.elapsed_us() / 3  # with the NTT, the gathers and the copies of the call
            m = re.search(r"k_unsatisfied_\w+", e.name)
            if m:
                us[m.group(0)] = us.get(m.group(0), 0.0) + e.time_range.elapsed_us() / 3
        size["device_us_per_prover_call"] = round(all_us, 1)
        size["kernel_us_per_call"] = {k: round(v, 1) for k, v in sorted(us.items())}
        size["kernel_ms_per_call_total"] = round(sum(us.values()) / 1e3, 3)
        result["sizes"]["2^%d" % log_n] = size
        del prover
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
