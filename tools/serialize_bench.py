"""Saving and reloading a compiled prover, on BenchCircuit<2^k> (the reference's benches/plonk.rs circuit):

  to_bytes      wall time of pb200_prover_to_bytes into a preallocated pageable buffer and the blob's GB/s;
                device time of its kernels (k_fr_to_canonical, k_poly_trim_len) from one further call traced by
                torch.profiler, and the kernels' GB/s over the 64 bytes they move per scalar
  reload        wall time of Prover.from_bytes(blob) beside Prover(...) = pb200_prover_new on the same circuit
  compress      pb200_g1_compress_batch on 2^20 points beside the per-point host loop (pb200_g1_compress) on a
                2^14-point sample, as ns per point

The two sides of a comparison alternate, --reps times each after one warm-up of each; times are the median and the
range of synchronous calls.  Needs a GPU; prints one JSON line with the card's name, power limit and maximum SM clock."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("k_fr_to_canonical", "k_poly_trim_len")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def stats(samples, scale=1e3, digits=2):
    s = sorted(samples)
    return {"median": round(s[len(s) // 2] * scale, digits), "range": [round(s[0] * scale, digits), round(s[-1] * scale, digits)]}


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="16,20")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--compress-log-points", type=int, default=20)
    a = ap.parse_args()

    import torch

    import plonk_b200
    from oracle import pyref as R
    from plonk_b200 import gadgets, kzg
    from plonk_b200._lib import check, lib

    if not torch.cuda.is_available():
        raise SystemExit("serialize_bench.py measures on a GPU and there is none")
    check(lib().pb200_init(0))
    result = {"card": card(), "reps": a.reps, "provers": []}
    srs = None
    for log_n in sorted((int(s) for s in a.log_n.split(",")), reverse=True):
        arr = gadgets.bench_circuit(1 << log_n).arrays()
        n_pts = (1 << (arr.constraints + 6 - 1).bit_length()) + 7
        if srs is None:  # the largest size comes first; smaller circuits take a prefix of its key
            buf = ctypes.create_string_buffer(96 * n_pts)
            check(lib().pb200_srs_setup_from_secret(R.fr_to_mont_bytes(0x1234567), R.fr_to_mont_bytes(0x7654321), n_pts, buf))
            srs = buf.raw

        def compile_():
            return plonk_b200.Prover(b"dusk-network", arr.constraints, arr.selectors, arr.wires, arr.n_witnesses, srs[: 96 * n_pts])

        prover = compile_()
        size = ctypes.c_size_t(prover.serialized_size())
        blob = ctypes.create_string_buffer(size.value)  # written in place: the C call is timed, not Python's copies

        def save():
            check(lib().pb200_prover_to_bytes(prover._h, blob, len(blob), ctypes.byref(size)))

        def reload_():
            return plonk_b200.Prover.from_bytes(blob, arr.wires, arr.n_witnesses)

        save()  # warm-up of to_bytes; also the reload's input
        assert reload_().commitments() == prover.commitments()  # warm-up of from_bytes
        t_save, t_load, t_new = [], [], []
        for _ in range(a.reps):
            t_save.append(timed(save)[0])
            dt, p = timed(reload_)
            t_load.append(dt)
            del p
            dt, p = timed(compile_)
            t_new.append(dt)
            del p
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            save()
        dev = {}
        for e in prof.key_averages():
            for k in KERNELS:
                if k in e.key:
                    dev[k] = round(dev.get(k, 0.0) + e.device_time_total / 1e3, 4)
        if "k_fr_to_canonical" not in dev:
            raise RuntimeError("the profiler trace does not hold k_fr_to_canonical")
        n = 1 << (arr.constraints - 1).bit_length()
        pk_scalars = (len(blob) - 48 - len(b"dusk-network") - 968 - 8 - 97 * n_pts - 16 - 15 * 8 - 17 * 172) // 32
        converted = pk_scalars - 8 * n  # the vanishing-polynomial evaluations are written by the host
        save = stats(t_save)
        row = {
            "circuit": "BenchCircuit<2^%d>" % log_n, "constraints": arr.constraints, "blob_bytes": len(blob),
            "to_bytes_wall_ms": save, "to_bytes_GBps": round(len(blob) / (save["median"] * 1e-3) / 1e9, 2),
            "to_bytes_device_ms": dev,
            "k_fr_to_canonical_GBps": round(64 * converted / (dev["k_fr_to_canonical"] * 1e-3) / 1e9, 1),
            "from_bytes_wall_ms": stats(t_load), "prover_new_wall_ms": stats(t_new),
        }
        row["reload_over_compile"] = round(row["from_bytes_wall_ms"]["median"] / row["prover_new_wall_ms"]["median"], 3)
        result["provers"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        del blob, prover

    n = 1 << a.compress_log_points
    buf = ctypes.create_string_buffer(96 * n)
    check(lib().pb200_srs_setup_from_secret(R.fr_to_mont_bytes(0x1234567), R.fr_to_mont_bytes(0x7654321), n, buf))
    pts = buf.raw
    sample = pts[: 96 << 14]
    out = ctypes.create_string_buffer(48 * n)
    one = ctypes.create_string_buffer(48)

    def batch():
        check(lib().pb200_g1_compress_batch(pts, n, out))

    def host_loop():
        L = lib()
        for i in range(0, len(sample), 96):
            L.pb200_g1_compress(sample[i : i + 96], one)

    batch()
    host_loop()
    assert out.raw[: 48 << 14] == b"".join(kzg.g1_compress(sample[i : i + 96]) for i in range(0, len(sample), 96))
    t_batch, t_host = [], []
    for _ in range(a.reps):
        t_batch.append(timed(batch)[0])
        t_host.append(timed(host_loop)[0])
    result["compress"] = {
        "batch_points": n, "batch_wall_ms": stats(t_batch), "batch_ns_per_point": round(sorted(t_batch)[len(t_batch) // 2] / n * 1e9, 2),
        "host_loop_points": 1 << 14, "host_loop_wall_ms": stats(t_host),
        "host_loop_ns_per_point": round(sorted(t_host)[len(t_host) // 2] / (1 << 14) * 1e9, 1),
        "note": "the host loop is timed through ctypes, one call per point, as the Python mirror made it",
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
