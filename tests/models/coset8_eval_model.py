"""Python model of k_coset8_eval + k_coset8_sum (plonk_b200/csrc/prover.cu): a polynomial's values on a coset
s*H_8 of the 8th roots of unity from one fold of its coefficients.

TEST INFRASTRUCTURE (like quotient_4n_model.py): restates the kernels' split of the work - blocks of groups of
eight coefficients, the groups of a thread, the lane, warp and block weights read from the same table of
y^(2^i) - so that the index algebra is checked against direct Horner evaluation.  Not on the product path.

With y = s^8 and F_r(y) = sum_q c_{8q+r} y^q (r < 8),

  f(s w8^k) = sum_r w8^(rk) s^r F_r(y),

an 8-point DFT of the eight folds.  Step 2 of the 4n-coset quotient needs the witness rows (n + 3 coefficients)
on h*H_8 and omega*h*H_8 and t mod (X^4n - g^4n) (4n coefficients) on h*H_8.

Run: python tests/models/coset8_eval_model.py"""
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import pyref as R  # noqa: E402

P = R.R_MOD

# the kernels' launch geometry: 256 threads of 32 lanes, 4 groups per thread in a full block, 32 block lanes
# per residue in the sum
KERNEL = dict(thread_bits=8, per=4, lane_bits=5, sum_lane_bits=5)


def consts(s, table_len=16):
    """Coset8Consts for one shift: s^r, y^(2^i)."""
    spow = [pow(s, r, P) for r in range(8)]
    ypow, y = [], pow(s, 8, P)
    for _ in range(table_len):
        ypow.append(y)
        y = y * y % P
    return spow, ypow


def weight(ypow, first, x, bits):
    """prod of ypow[first + k] over the set bits k < bits of x: y^(x 2^first)"""
    w = 1
    for k in range(bits):
        if x >> k & 1:
            w = w * ypow[first + k] % P
    return w


def coset8_eval(c, s, w8, thread_bits, per, lane_bits, sum_lane_bits):
    """f(s w8^k), k < 8, computed the way the two kernels split it."""
    threads = 1 << thread_bits
    block_bits = thread_bits + (per.bit_length() - 1)
    assert per == 1 << (block_bits - thread_bits)
    spow, ypow = consts(s, block_bits + sum_lane_bits + 1)
    groups = (len(c) + 7) // 8
    nb = max(1, groups >> block_bits)
    coef = lambda k: c[k] if k < len(c) else 0
    partial = []
    # k_coset8_eval: one CTA per block
    for b in range(nb):
        end = groups if b + 1 == nb else (b + 1) << block_bits
        warp_sums = {}
        for t in range(threads):
            g0 = (b << block_bits) + t
            top = (end - 1 - g0) // threads if g0 < end else -1
            acc = [coef(8 * (g0 + threads * top) + r) if top >= 0 else 0 for r in range(8)]
            for i in range(top - 1, -1, -1):
                acc = [(acc[r] * ypow[thread_bits] + coef(8 * (g0 + threads * i) + r)) % P for r in range(8)]
            lane, warp = t & ((1 << lane_bits) - 1), t >> lane_bits
            w = weight(ypow, 0, lane, lane_bits)
            ws = warp_sums.setdefault(warp, [0] * 8)
            for r in range(8):
                ws[r] = (ws[r] + acc[r] * w) % P
        blk = [0] * 8
        for warp, ws in warp_sums.items():
            w = weight(ypow, lane_bits, warp, thread_bits - lane_bits)
            for r in range(8):
                blk[r] = (blk[r] + ws[r] * w) % P
        partial.append(blk)
    # k_coset8_sum: block lane p takes blocks p, p + 32, ... with weights Z^b, Z = y^(2^block_bits)
    F = [0] * 8
    for p in range(1 << sum_lane_bits):
        w = weight(ypow, block_bits, p, sum_lane_bits)
        for b in range(p, nb, 1 << sum_lane_bits):
            for r in range(8):
                F[r] = (F[r] + partial[b][r] * w) % P
            w = w * ypow[block_bits + sum_lane_bits] % P
    g = [F[r] * spow[r] % P for r in range(8)]
    return [sum(g[r] * pow(w8, r * k % 8, P) for r in range(8)) % P for k in range(8)]


def check(log_n, seed, geometry=KERNEL):
    """Rows of n + 3 and the 4n polynomial on both cosets of step 2 against Horner at the 16 points."""
    rng = random.Random(seed)
    n = 1 << log_n
    w8n, wn = R.EvaluationDomain(8 * n).group_gen, R.EvaluationDomain(n).group_gen
    h, w8 = R.GENERATOR * w8n % P, pow(w8n, n, P)
    for length in (n + 3, 4 * n):
        c = [rng.randrange(P) for _ in range(length)]
        for s in (h, h * wn % P):
            got = coset8_eval(c, s, w8, **geometry)
            want = [R.poly_eval(c, s * pow(w8, k, P) % P) for k in range(8)]
            assert got == want, (log_n, length, geometry)


if __name__ == "__main__":
    for log_n in range(4, 11):
        check(log_n, log_n)
        check(log_n, log_n, dict(thread_bits=2, per=2, lane_bits=1, sum_lane_bits=5))
        print(f"n = 2^{log_n}: fold + DFT == Horner at the 16 points")
    print("ok")
