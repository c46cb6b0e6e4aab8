"""Times Circuit::compress (plonk_b200.compress_arrays, host) and Compiler::compile_with_compressed against
Compiler::compile for the reference's BenchCircuit<2^16> and <2^20>, with the card's name and power limit read in the
same run.  Prints one JSON object; --out also writes it to a file outside the tree.

compile and compile_with_compressed are alternated round by round on one set of public parameters; each time covers the
whole call (decoding or the column export, preprocessing on the GPU, the Verifier).  compress is timed on the arrays the
native composer exported, so the circuit's synthesis is not in it.

    python tools/compress_bench.py --rounds 3 --out /tmp/compress_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # a machine without nvidia-smi still gets its times
        return {"gpu": "unknown (%s)" % e}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-sizes", default="16,20")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import plonk_b200
    from plonk_b200 import gadgets

    plonk_b200.lib().pb200_init(0)
    mont = lambda v: (v * (1 << 256) % 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001).to_bytes(32, "little")
    result = {"info": gpu_info(), "sizes": {}}
    for log_n in (int(x) for x in args.log_sizes.split(",")):
        comp = gadgets.bench_circuit(1 << log_n)
        arrays = comp.arrays()
        pp = plonk_b200.PublicParameters.setup((1 << (log_n + 1)) + 6, [mont(v) for v in (0x1234567, 0x7654321, 0xABCDEF)])
        label = b"compress-bench"
        t_compress, t_direct, t_compressed = [], [], []
        data = b""
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            data = plonk_b200.compress_arrays(arrays)
            t_compress.append(time.perf_counter() - t0)
        plonk_b200.Compiler.compile_with_compressed(pp, label, data)  # warm-up: twiddles, tables, pools
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            p, v = plonk_b200.Compiler.compile(pp, label, comp)
            t_direct.append(time.perf_counter() - t0)
            del p, v
            t0 = time.perf_counter()
            p, v = plonk_b200.Compiler.compile_with_compressed(pp, label, data)
            t_compressed.append(time.perf_counter() - t0)
            del p, v
        ms = lambda xs: {"median_ms": round(1e3 * statistics.median(xs), 2), "min_ms": round(1e3 * min(xs), 2)}
        result["sizes"]["2^%d" % log_n] = {
            "constraints": arrays.constraints, "compressed_bytes": len(data), "compress": ms(t_compress),
            "compile": ms(t_direct), "compile_with_compressed": ms(t_compressed), "rounds": args.rounds,
        }
    text = json.dumps(result)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
