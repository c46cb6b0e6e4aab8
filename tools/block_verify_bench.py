"""Batch verification of a block holding proofs of K circuits on one SRS: one pb200_batch_verify_groups call against
K pb200_batch_verify calls one after another and against K threads making one pb200_batch_verify call each, for
K in 1, 2, 4, 8 and N = 16, 256, 4096 proofs in total.

The circuits are BenchCircuit<2^16>, <2^15>, <2^14> and <2^13> (the reference's benches/plonk.rs circuit) and four
synthetic arithmetic circuits of 2^12 gates, all on one SRS with known secrets; the first K make a block.  64 distinct
V3 proofs are made per circuit with the GPU prover and tiled to N / K per group.  Before timing, every form must accept
every block, and a block with one tampered proof in its last group must fail the grouped call.  In one process the
three forms alternate, --reps times each per (K, N), after a warm-up of each; wall time is the median of synchronous
calls, with its range.  Per-kernel device ms come from one further call of each form, traced by torch.profiler (CUDA
activities) in a run of its own.  Prints one JSON line with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.batch_verify_bench import KERNELS, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--totals", default="16,256,4096")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()

    import torch

    import plonk_b200
    from oracle import cref
    from oracle import pyref as R
    from plonk_b200 import gadgets
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    draws = [R.fr_to_mont_bytes(v) for v in (0x1234567, 0x7654321, 0xABCDEF)]  # one SRS: every circuit shares its opening key
    arrays = [(b"dusk-network", gadgets.bench_circuit(1 << log_n).arrays()) for log_n in (16, 15, 14, 13)]
    for seed in range(4):
        comp = R.Composer.initialized()
        R.synthetic_arith_circuit(comp, (1 << 12) - 12, seed=400 + seed, n_public=3, widgets=9)
        arrays.append((b"block-synthetic-%d" % seed, cref.CircuitArrays(comp)))
    max_k = max(int(s) for s in a.ks.split(","))
    circuits = []
    for label, arr in arrays[:max_k]:
        n = 1 << (arr.constraints + 6 - 1).bit_length()
        pp = plonk_b200.PublicParameters.setup(n, draws)
        prover, verifier = plonk_b200.Compiler.compile(pp, label, SimpleNamespace(arrays=lambda arr=arr: arr))
        proofs = [prover.prove(arr.witnesses, arr.pi_idx, arr.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(s))) for s in range(64)]
        del prover
        circuits.append((verifier, proofs, arr.pi_vals, arr.constraints))
    pool = ThreadPoolExecutor(max_workers=max_k)

    def block(k, total):
        per = total // k
        return [(v, [ps[(g * 7 + i) % 64] for i in range(per)], [pi] * per, plonk_b200.PlonkVersion.V3)
                for g, (v, ps, pi, _) in enumerate(circuits[:k])]

    def grouped(groups):
        plonk_b200.batch_verify_groups(groups)

    def sequential(groups):
        for v, ps, pis, ver in groups:
            v.batch_verify(ps, pis, ver)

    def threads(groups):
        for f in [pool.submit(v.batch_verify, ps, pis, ver) for v, ps, pis, ver in groups]:
            f.result()

    forms = (("groups", grouped), ("sequential", sequential), ("threads", threads))
    rows = []
    for k in [int(s) for s in a.ks.split(",")]:
        for total in [int(s) for s in a.totals.split(",")]:
            groups = block(k, total)
            for _, fn in forms:
                fn(groups)  # every form accepts the block; also the warm-up of this shape
            v, ps, pis, ver = groups[-1]
            bad = list(ps)
            tampered = bytearray(bad[-1])
            tampered[528 + 7] ^= 1
            bad[-1] = bytes(tampered)
            try:
                grouped(groups[:-1] + [(v, bad, pis, ver)])
                raise AssertionError("a block with a tampered proof was accepted")
            except plonk_b200.ProofVerificationError:
                pass
            walls = {m: [] for m, _ in forms}
            for _ in range(a.reps):
                for m, fn in forms:
                    t = time.perf_counter()
                    fn(groups)
                    walls[m].append(time.perf_counter() - t)
            row = {"k": k, "n": total}
            for m, _ in forms:
                w = sorted(walls[m])
                row[m + "_wall_ms"] = round(w[len(w) // 2] * 1e3, 3)
                row[m + "_wall_ms_range"] = [round(w[0] * 1e3, 3), round(w[-1] * 1e3, 3)]
            for m, fn in forms:
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                    fn(groups)
                dev = {}
                for e in prof.key_averages():
                    for name in KERNELS:
                        if name in e.key:
                            dev[name] = round(dev.get(name, 0.0) + e.device_time_total / 1e3, 4)
                if not dev:
                    raise RuntimeError("the profiler trace holds none of the verifier's kernels")
                row[m + "_device_ms"] = dev
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    pool.shutdown()
    names = ["%s(%d rows)" % (label.decode(), c[3]) for (label, _), c in zip(arrays, circuits)]
    print(json.dumps({"card": card(), "circuits": names, "reps": a.reps, "rows": rows}))


if __name__ == "__main__":
    main()
