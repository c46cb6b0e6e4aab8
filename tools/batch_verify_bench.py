"""Batch verification against per-proof verification on BenchCircuit<2^16> proofs (the reference's benches/plonk.rs
circuit): pb200_batch_verify (one verdict, one pairing) against pb200_verify (one verdict and one pairing per proof), at
batch sizes 1, 16, 256, 4096 and 16384.

64 distinct proofs are made with the GPU prover and tiled to the batch size.  Before timing, both calls must accept
every batch, and a batch with one tampered proof must fail the batch call.  In one process the two calls alternate,
--reps times each per batch size, after a warm-up of each; wall time is the median of synchronous calls.  Per-kernel
device ms come from one further call of each, traced by torch.profiler (CUDA activities) in a run of its own.  Prints
one JSON line with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("k_g1_decompress", "k_verify_msm", "k_verify_pairing", "k_batch_fold", "k_batch_key_sums", "k_batch_msm", "k_batch_reduce")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=16)
    ap.add_argument("--batches", default="1,16,256,4096,16384")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()

    import torch

    import plonk_b200
    from oracle import pyref as R
    from oracle import cref
    from plonk_b200 import gadgets
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    comp = gadgets.bench_circuit(1 << a.log_n)
    arr = comp.arrays()
    n = 1 << (arr.constraints + 6 - 1).bit_length()
    pp = plonk_b200.PublicParameters.setup(n, [R.fr_to_mont_bytes(v) for v in (0x1234567, 0x7654321, 0xABCDEF)])
    prover, verifier = plonk_b200.Compiler.compile(pp, b"dusk-network", comp)
    proofs = [prover.prove(arr.witnesses, arr.pi_idx, arr.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(s))) for s in range(64)]
    bad = bytearray(proofs[5])
    bad[528 + 7] ^= 1
    try:
        verifier.batch_verify(proofs[:5] + [bytes(bad)] + proofs[6:16], [arr.pi_vals] * 16)
        raise AssertionError("a batch with a tampered proof was accepted")
    except plonk_b200.ProofVerificationError:
        pass

    def per_proof(batch, pb):
        assert verifier.verify_batch(batch, pb) == [0] * len(batch)

    def batched(batch, pb):
        verifier.batch_verify(batch, pb)

    modes = (("verify", per_proof), ("batch_verify", batched))
    rows = []
    for b in [int(s) for s in a.batches.split(",")]:
        batch = [proofs[i % 64] for i in range(b)]
        pb = [arr.pi_vals] * b
        walls = {m: [] for m, _ in modes}
        for _, fn in modes:
            fn(batch, pb)  # warm-up of this shape
        for _ in range(a.reps):
            for m, fn in modes:
                t = time.perf_counter()
                fn(batch, pb)
                walls[m].append(time.perf_counter() - t)
        row = {"batch": b}
        for m, fn in modes:
            wall = sorted(walls[m])[len(walls[m]) // 2]
            row[m + "_wall_ms"] = round(wall * 1e3, 3)
            row[m + "_wall_ms_range"] = [round(min(walls[m]) * 1e3, 3), round(max(walls[m]) * 1e3, 3)]
        for m, fn in modes:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn(batch, pb)
            dev = {}
            for e in prof.key_averages():
                for k in KERNELS:
                    if k in e.key:
                        dev[k] = round(dev.get(k, 0.0) + e.device_time_total / 1e3, 4)
            if not dev:
                raise RuntimeError("the profiler trace holds none of the verifier's kernels")
            row[m + "_device_ms"] = dev
        row["speedup"] = round(row["verify_wall_ms"] / row["batch_verify_wall_ms"], 3)
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps({"card": card(), "circuit": "BenchCircuit<2^%d>" % a.log_n, "reps": a.reps, "rows": rows}))


if __name__ == "__main__":
    main()
