"""Verified proofs per second of the GPU Verifier on BenchCircuit<2^16> proofs (the reference's benches/plonk.rs
circuit), at batch sizes 1, 16, 256 and 4096, split into host and device milliseconds per proof.

64 distinct proofs are made with the GPU prover and tiled to the batch size.  Before timing, every one of them must
be accepted and a batch with one tampered proof must reject exactly that one.  Wall time is the median of --reps
synchronous calls.  Device ms is the summed time of the library's kernels in one further call traced by
torch.profiler (CUDA activities); host ms is wall minus device: the transcript replays, the scalar algebra and the
copies.  Prints one JSON line with the card's name, power limit and maximum SM clock.  Needs an H100; there is no
CPU baseline here (the reference quotes 2.8 ms per proof on its CPU; that figure is not measured here)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    ap.add_argument("--batches", default="1,16,256,4096")
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
    pis = [arr.pi_vals] * 64
    assert verifier.verify_batch(proofs, pis) == [0] * 64, "a valid proof was rejected"
    bad = bytearray(proofs[5])
    bad[528 + 7] ^= 1
    got = verifier.verify_batch(proofs[:5] + [bytes(bad)] + proofs[6:16], pis[:16])
    assert got == [0] * 5 + [plonk_b200._lib.PB200_ERR_VERIFY] + [0] * 10, got

    rows = []
    for b in [int(s) for s in a.batches.split(",")]:
        batch = [proofs[i % 64] for i in range(b)]
        pb = [arr.pi_vals] * b
        verifier.verify_batch(batch, pb)  # warm-up of this shape
        walls = []
        for _ in range(a.reps):
            t = time.perf_counter()
            st = verifier.verify_batch(batch, pb)
            walls.append(time.perf_counter() - t)
        assert st == [0] * b
        wall = sorted(walls)[len(walls) // 2]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            verifier.verify_batch(batch, pb)
        kernels = ("k_g1_decompress", "k_verify_msm", "k_verify_pairing")
        dev_us = sum(e.device_time_total for e in prof.key_averages() if any(k in e.key for k in kernels))
        if dev_us <= 0:
            raise RuntimeError("the profiler trace holds none of the verifier's kernels")
        dev_ms = dev_us / 1e3
        rows.append({"batch": b, "proofs_per_s": round(b / wall, 1), "wall_ms_per_proof": round(wall * 1e3 / b, 4),
                     "device_ms_per_proof": round(dev_ms / b, 4), "host_ms_per_proof": round(max(0.0, wall * 1e3 - dev_ms) / b, 4)})
    print(json.dumps({"card": card(), "circuit": "BenchCircuit<2^%d>" % a.log_n, "rows": rows,
                      "note": "host = wall - device kernel time; reference CPU figure 2.8 ms/proof is the reference's own, not measured here"}))


if __name__ == "__main__":
    main()
