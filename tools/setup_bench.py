"""Times PublicParameters::setup on the GPU (pb200_public_parameters_setup) and its commit-key kernel
(pb200_srs_setup_from_secret) at 2^16, 2^20 and 2^24 points (+7), with the card's name and power limit read in the same
run.

For a same-run A/B against another build of the library (say the parent commit's, built with
`PB200_SRC=<its csrc> PB200_OUT=<path> ./build.sh`, INTEGRATION.md section 7), pass --baseline-lib <path>: each round
runs one process per library, alternating, and each process loads its library through PB200_LIB.  A library without
pb200_public_parameters_setup is timed on pb200_srs_setup_from_secret only.

Times are host wall clock around the synchronous call: the kernel, the generator table's lazy build excluded by a
warm-up call, and the device-to-host copy of the points (96 bytes each) that every caller pays.

    python tools/setup_bench.py --rounds 3 --baseline-lib /path/to/parent/libplonk_b200.so --out setup_bench.json
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_MOD = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
DRAWS = (0x1234567, 0x7654321, 0xABCDEF)  # x, g_scalar, h_scalar


def mont(v: int) -> bytes:
    return (v * (1 << 256) % R_MOD).to_bytes(32, "little")


def worker(log_sizes, reps: int) -> dict:
    """One library (the one PB200_LIB names, else the tree's): median and min call time per size."""
    sys.path.insert(0, ROOT)
    from plonk_b200._lib import LIB_PATH

    L = ctypes.CDLL(LIB_PATH)
    L.pb200_srs_setup_from_secret.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    has_pp = hasattr(L, "pb200_public_parameters_setup")
    if has_pp:
        L.pb200_public_parameters_setup.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 5
    L.pb200_last_error.restype = ctypes.c_char_p

    def ok(rc):
        if rc != 0:
            raise RuntimeError(f"error {rc}: {L.pb200_last_error().decode()}")

    ok(L.pb200_init(0))
    x, gs, hs = (mont(v) for v in DRAWS)
    out = {"lib": LIB_PATH, "sizes": {}}
    okey = ctypes.create_string_buffer(240)
    for log_n in log_sizes:
        n = (1 << log_n) + 7
        buf = ctypes.create_string_buffer(96 * n)
        row = {}
        calls = {"commit_key": lambda: ok(L.pb200_srs_setup_from_secret(x, gs, n, buf))}
        if has_pp:
            calls["public_parameters"] = lambda: ok(L.pb200_public_parameters_setup(n - 7, x, gs, hs, buf, okey))
        for name, call in calls.items():
            call()  # warm-up: module load, the generator table, host pages of the output
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                call()
                ts.append((time.perf_counter() - t0) * 1e3)
            row[name] = {"median_ms": statistics.median(ts), "min_ms": min(ts), "all_ms": ts}
        row["first_point_hex"] = buf.raw[:96].hex()
        row["last_point_hex"] = buf.raw[96 * (n - 1) : 96 * n].hex()
        out["sizes"][str(log_n)] = row
        del buf
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-sizes", default="16,20,24")
    ap.add_argument("--reps", type=int, default=3, help="timed calls per size in one process (median reported)")
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the libraries (spread across processes)")
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    sizes = [int(s) for s in a.log_sizes.split(",")]
    if a.worker:
        print(json.dumps(worker(sizes, a.reps)))
        return
    libs = {"new": os.path.join(ROOT, "plonk_b200", "libplonk_b200.so")}
    if a.baseline_lib:
        libs["baseline"] = os.path.abspath(a.baseline_lib)
    result = {"card": card(), "draws": [hex(d) for d in DRAWS], "rounds": []}
    for r in range(a.rounds):
        rnd = {}
        for tag, path in libs.items():
            env = dict(os.environ, PB200_LIB=path)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--log-sizes", a.log_sizes, "--reps", str(a.reps)],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"{tag} worker failed:\n{p.stdout}\n{p.stderr}")
            rnd[tag] = json.loads(p.stdout.strip().splitlines()[-1])
            for log_n, row in rnd[tag]["sizes"].items():
                times = "  ".join(f"{k} {v['median_ms']:.2f} ms" for k, v in row.items() if isinstance(v, dict))
                print(f"round {r} {tag:8s} 2^{log_n}+7: {times}", flush=True)
        if "baseline" in rnd:  # same draws, same points
            for log_n, row in rnd["new"]["sizes"].items():
                base = rnd["baseline"]["sizes"][log_n]
                assert (row["first_point_hex"], row["last_point_hex"]) == (base["first_point_hex"], base["last_point_hex"]), log_n
        result["rounds"].append(rnd)
    summary = {}
    for tag in libs:
        for log_n in (str(s) for s in sizes):
            for name in ("commit_key", "public_parameters"):
                v = [rnd[tag]["sizes"][log_n][name]["median_ms"] for rnd in result["rounds"] if name in rnd[tag]["sizes"][log_n]]
                if v:
                    summary[f"{tag} {name} 2^{log_n}+7"] = {"median_of_rounds_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
    result["summary"] = summary
    print(json.dumps({"card": result["card"], "summary": summary}, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
