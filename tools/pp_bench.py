"""Times DevicePublicParameters against PublicParameters on the GPU, with the card's name, power limit and maximum SM
clock read in the same run.  Prints one JSON line (and writes it to --out when given).

For BenchCircuit<2^16> and <2^20> (--log-sizes), in one process:
  * compile: Compiler.compile from the host pp, against the first and the second compile from one fresh device pp of
    two different circuits of that size (the BenchCircuit, then a seeded arithmetic circuit with the same gate count,
    so the same domain and trimmed key);
  * from_bytes: Prover.from_bytes of the BenchCircuit prover's bytes without and with the device pp (whose tables are
    already built);
  * memory: device bytes (torch.cuda.mem_get_info, after a synchronise) taken by one more prover of the BenchCircuit
    from the host pp and from the device pp that already holds its tables.
And at --setup-log-sizes (2^20, 2^24 powers): PublicParameters.setup / from_slice against DevicePublicParameters.setup
/ from_slice.

Each measurement alternates the forms it compares, --rounds times, after a warm-up of every form; medians with the
min-max range are reported.  Times are host wall clock around synchronous calls (every call here synchronises).

    python tools/pp_bench.py --rounds 3 --out pp_bench.json
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R_MOD = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
DRAWS = (0x1234567, 0x7654321, 0xABCDEF)  # x, g_scalar, h_scalar
LABEL = b"pp-bench"


def mont(v: int) -> bytes:
    return (v * (1 << 256) % R_MOD).to_bytes(32, "little")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def summary(ts) -> dict:
    return {"median": statistics.median(ts), "min": min(ts), "max": max(ts), "all": ts}


def timed(call):
    t0 = time.perf_counter()
    out = call()
    return (time.perf_counter() - t0) * 1e3, out


def arith_composer(gates: int, seed: int):
    """A seeded circuit of arithmetic gates only, exactly `gates` long."""
    from plonk_b200 import gadgets as N

    c = N.Composer.initialized()
    rng = random.Random(seed)
    acc = c.append_witness(rng.randrange(R_MOD))
    while c.constraints() < gates:
        acc = c.gate_add(dict(q_l=rng.randrange(1, 1 << 20), q_r=rng.randrange(1, 1 << 20)), a=acc, b=c.append_witness(rng.randrange(R_MOD)))
    return c


def compile_bench(log_n: int, host_pp, rounds: int, torch) -> dict:
    import plonk_b200
    from plonk_b200 import gadgets as N
    from plonk_b200._lib import check, lib

    bench = N.bench_circuit(1 << log_n)
    other = arith_composer(bench.constraints(), log_n)
    arrays = bench.arrays()
    C, D = plonk_b200.Compiler, plonk_b200.DevicePublicParameters

    def free_bytes():
        check(lib().pb200_device_sync())
        return torch.cuda.mem_get_info()[0]

    # warm-up: every form once (modules, the stream pool at this size)
    C.compile(host_pp, LABEL, bench)
    warm = D.from_host(host_pp)
    C.compile(warm, LABEL, bench)
    blob = C.compile(host_pp, LABEL, bench)[0].to_bytes()
    plonk_b200.Prover.from_bytes(blob, arrays.wires, arrays.n_witnesses, pp=warm)
    gc.collect()
    host, first, second, load_plain, load_pp = [], [], [], [], []
    for _ in range(rounds):
        t, _ = timed(lambda: C.compile(host_pp, LABEL, bench))
        host.append(t)
        gc.collect()
        dpp = D.from_host(host_pp)
        t1, p1 = timed(lambda: C.compile(dpp, LABEL, bench))
        t2, p2 = timed(lambda: C.compile(dpp, LABEL, other))
        first.append(t1)
        second.append(t2)
        t, _ = timed(lambda: plonk_b200.Prover.from_bytes(blob, arrays.wires, arrays.n_witnesses))
        load_plain.append(t)
        gc.collect()
        t, _ = timed(lambda: plonk_b200.Prover.from_bytes(blob, arrays.wires, arrays.n_witnesses, pp=dpp))
        load_pp.append(t)
        del p1, p2, dpp
        gc.collect()
    # memory of one more prover: a host-pp prover builds its own tables, a device-pp one shares the pp's
    keep = [C.compile(host_pp, LABEL, bench)]
    before = free_bytes()
    keep.append(C.compile(host_pp, LABEL, bench))
    host_bytes = before - free_bytes()
    dpp = D.from_host(host_pp)
    keep.append(C.compile(dpp, LABEL, bench))
    before = free_bytes()
    keep.append(C.compile(dpp, LABEL, other))
    shared_bytes = before - free_bytes()
    tables = dpp.tables()
    return {
        "constraints": bench.constraints(),
        "compile_host_pp_ms": summary(host),
        "compile_device_pp_first_ms": summary(first),
        "compile_device_pp_second_ms": summary(second),
        "from_bytes_ms": summary(load_plain),
        "from_bytes_device_pp_ms": summary(load_pp),
        "bytes_per_extra_prover_host_pp": host_bytes,
        "bytes_per_extra_prover_device_pp": shared_bytes,
        "device_pp_tables": tables._asdict(),
    }


def setup_bench(log_d: int, rounds: int) -> dict:
    import plonk_b200

    draws = [mont(v) for v in DRAWS]
    P, D = plonk_b200.PublicParameters, plonk_b200.DevicePublicParameters
    d = 1 << log_d
    host = P.setup(d, draws)  # warm-up of both forms, and the bytes from_slice reads
    D.setup(d, draws)
    data = host.to_var_bytes()
    del host
    P.from_slice(data)
    D.from_slice(data)
    gc.collect()
    out = {k: [] for k in ("setup_host_ms", "setup_device_ms", "from_slice_host_ms", "from_slice_device_ms")}
    for _ in range(rounds):
        for key, call in (("setup_host_ms", lambda: P.setup(d, draws)), ("setup_device_ms", lambda: D.setup(d, draws)),
                          ("from_slice_host_ms", lambda: P.from_slice(data)), ("from_slice_device_ms", lambda: D.from_slice(data))):
            t, obj = timed(call)
            out[key].append(t)
            del obj
            gc.collect()
    return {"points": d + 7, **{k: summary(v) for k, v in out.items()}}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-sizes", default="16,20")
    ap.add_argument("--setup-log-sizes", default="20,24")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    import plonk_b200
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    torch.cuda.init()
    result = {"card": card(), "compile": {}, "setup": {}}
    sizes = [int(s) for s in a.log_sizes.split(",") if s]
    if sizes:
        host_pp = plonk_b200.PublicParameters.setup(1 << max(sizes), [mont(v) for v in DRAWS])
        for log_n in sizes:
            result["compile"][str(log_n)] = compile_bench(log_n, host_pp, a.rounds, torch)
        del host_pp
        gc.collect()
    for log_d in [int(s) for s in a.setup_log_sizes.split(",") if s]:
        result["setup"][str(log_d)] = setup_bench(log_d, a.rounds)
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
