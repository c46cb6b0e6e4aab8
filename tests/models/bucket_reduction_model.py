"""Schedule of the MSM bucket reduction (csrc/msm.cu: k_msm_rows_cols, k_msm_lists, k_msm_fold, k_msm_final and the
host Horner of msm_finish), replayed on an abstract group so that it can be checked against R = sum_b (b + 1) B_b.

The bucket index is written b = g G + j (g = 8 buckets per row G, column j < g):
    R = sum_j (j + 1) T_j + g sum_G G S_G,   T_j = sum_G B[gG + j] (column sums),   S_G = sum_j B[gG + j] (row sums)
The kernels leave [ndig + 1] digit sums: D_j = sum_v v C_{j,v}, where C_{j,v} is the sum of the S_G whose digit j
(plan.bits[j] bits from plan.shift[j]) equals v, and sum_j (j + 1) T_j last.  The host adds them by
Horner: R = D_ndig + g sum_j 2^shift_j D_j.  The model follows the kernels' index arithmetic (member enumeration
of a class, column partial layout, chunking, suffix scans) and counts the full additions and the longest chain of
dependent ones, so that a change of the schedule is checked here before it is written in CUDA."""

K_GROUP, K_COL_RUN, K_LIST_CHUNK, K_FINAL_CHUNKS = 8, 8, 256, 4


class IntGroup:
    """Z/r with (value, depth): depth = dependent additions that produced the value."""
    r = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001

    def __init__(self):
        self.adds = 0

    zero = (0, 0, True)  # (value, depth, is identity)

    def add(self, a, b):
        if a[2]:
            return b
        if b[2]:
            return a
        self.adds += 1
        return ((a[0] + b[0]) % self.r, max(a[1], b[1]) + 1, False)

    def dbl_times(self, a, k):  # host doublings: not counted
        return ((a[0] << k) % self.r, a[1], a[2])

    def point(self, v):
        return (v % self.r, 0, False)


def plan_for(c):
    """msm_plan_c"""
    nb = 1 << (c - 1)
    g = min(K_GROUP, nb)
    n_groups = nb // g
    log_g = g.bit_length() - 1
    total_bits = (n_groups - 1).bit_length() if n_groups > 1 else 0
    ndig = (total_bits + 3) // 4
    assert ndig <= 7
    shift, bits, first_class = [], [], []
    sh = cls = 0
    for j in range(ndig):
        b = (total_bits - sh) // (ndig - j)
        shift.append(sh)
        bits.append(b)
        first_class.append(cls)
        sh += b
        cls += 1 << b
    return {"nb": nb, "g": g, "n_groups": n_groups, "log_g": log_g, "ndig": ndig, "shift": shift, "bits": bits,
            "first_class": first_class, "n_digit_classes": cls, "n_columns": g, "nlists": cls + g}


def warp_sum(G, vals):
    """shfl_down tree over 32 lanes (d = 16 .. 1): lane 0's result.  Only the additions that reach lane 0 are
    modelled (and counted); the other lanes of the warp compute values nobody reads."""
    v = list(vals)
    d = 16
    while d:
        v = [G.add(v[i], v[i + d]) if i < d else v[i] for i in range(32)]
        d >>= 1
    return v[0]


def weighted_lane_sum(G, x, n, first):
    """sum_{k >= first} (k + 1 - first) x_k over lanes k < n (inclusive suffix scan, then a tree over lanes first..n-1)"""
    x = list(x) + [G.zero] * (32 - len(x))
    d = 1
    while d < n:
        x = [G.add(x[i], x[i + d]) if i + d < n else x[i] for i in range(32)]
        d <<= 1
    y = [x[i] if first <= i < n else G.zero for i in range(32)]
    d = n >> 1
    while d:
        y = [G.add(y[i], y[i + d]) if i < d else y[i] for i in range(32)]
        d >>= 1
    return y[0]


def reduce(G, buckets, c):
    """The device kernels and the host Horner; returns R."""
    p = plan_for(c)
    nb, g, n_groups = p["nb"], p["g"], p["n_groups"]
    assert len(buckets) == nb
    col_run = min(K_COL_RUN, n_groups)
    n_parts = n_groups // col_run
    # A. k_msm_rows_cols
    S = []
    for t in range(n_groups):
        acc = G.zero
        for j in range(g):
            acc = G.add(acc, buckets[t * g + j])
        S.append(acc)
    P = [[None] * n_parts for _ in range(g)]
    for u in range(g * n_parts):
        j, part = divmod(u, n_parts)
        acc = G.zero
        for k in range(col_run):
            acc = G.add(acc, buckets[(part * col_run + k) * g + j])
        P[j][part] = acc
    # B. k_msm_lists
    chunks = max([(n_parts + K_LIST_CHUNK - 1) // K_LIST_CHUNK] +
                 [((n_groups >> b) + K_LIST_CHUNK - 1) // K_LIST_CHUNK for b in p["bits"]] + [1])
    lists = [[G.zero] * chunks for _ in range(p["nlists"])]
    for lst in range(p["nlists"]):
        for chunk in range(chunks):
            lanes = [G.zero] * 32
            if lst < p["n_digit_classes"]:
                j = 0
                while j + 1 < p["ndig"] and lst >= p["first_class"][j + 1]:
                    j += 1
                v = lst - p["first_class"][j]
                sh, bits = p["shift"][j], p["bits"][j]
                count = n_groups >> bits
                for lane in range(32):
                    for idx in range(chunk * K_LIST_CHUNK + lane, min(count, (chunk + 1) * K_LIST_CHUNK), 32):
                        Gi = ((idx >> sh) << (sh + bits)) | (v << sh) | (idx & ((1 << sh) - 1))
                        lanes[lane] = G.add(lanes[lane], S[Gi])
            else:
                col = lst - p["n_digit_classes"]
                for lane in range(32):
                    for idx in range(chunk * K_LIST_CHUNK + lane, min(n_parts, (chunk + 1) * K_LIST_CHUNK), 32):
                        lanes[lane] = G.add(lanes[lane], P[col][idx])
            lists[lst][chunk] = warp_sum(G, lanes)
    if chunks > K_FINAL_CHUNKS:  # k_msm_fold
        folded = []
        for lst in range(p["nlists"]):
            lanes = [G.zero] * 32
            for k in range(chunks):
                lanes[k % 32] = G.add(lanes[k % 32], lists[lst][k])
            folded.append([warp_sum(G, lanes)])
        lists, chunks = folded, 1
    # C. k_msm_final
    out = []
    for w in list(range(p["ndig"])) + [7]:
        digit = w < p["ndig"]
        n = (1 << p["bits"][w]) if digit else p["n_columns"]
        first_list = p["first_class"][w] if digit else p["n_digit_classes"]
        x = []
        for lane in range(n):
            acc = G.zero
            for ch in range(chunks):
                acc = G.add(acc, lists[first_list + lane][ch])
            x.append(acc)
        out.append(weighted_lane_sum(G, x, n, 1 if digit else 0))
    depth = max(o[1] for o in out)
    # msm_finish: Horner over the digits, then the column part
    h = G.zero
    for d in range(p["ndig"] - 1, -1, -1):
        h = G.add(h, out[d])
        h = G.dbl_times(h, p["bits"][d - 1] if d > 0 else p["log_g"])
    h = G.add(h, out[p["ndig"]])
    return h, depth


def check(c, seed=0, density=1.0):
    import random

    rng = random.Random(seed)
    G = IntGroup()
    nb = 1 << (c - 1)
    buckets = [G.point(rng.randrange(1, G.r)) if rng.random() < density else G.zero for _ in range(nb)]
    want = sum((b + 1) * v[0] for b, v in enumerate(buckets) if not v[2]) % G.r
    got, depth = reduce(G, buckets, c)
    assert (got[0] if not got[2] else 0) == want, f"c = {c}: reduction differs from sum (b + 1) B_b"
    return G.adds, depth


def check_curve(c, seed=0):
    """The same schedule on BLS12-381 G1 points (oracle Jacobian arithmetic) for a small window."""
    import random

    from oracle import pyref as R

    class CurveGroup:
        zero = (None, 0, True)

        def add(self, a, b):
            if a[2]:
                return b
            if b[2]:
                return a
            s = R.jac_add(a[0], b[0])
            return (s, max(a[1], b[1]) + 1, False)

        def dbl_times(self, a, k):
            if a[2]:
                return a
            v = a[0]
            for _ in range(k):
                v = R.jac_double(v)
            return (v, a[1], False)

    rng = random.Random(seed)
    nb = 1 << (c - 1)
    ks = [rng.randrange(1, R.R_MOD) if rng.random() < 0.8 else 0 for _ in range(nb)]
    G = CurveGroup()
    buckets = [(R.jac_from_affine(R.g1_mul(R.G1_GEN, k)), 0, False) if k else G.zero for k in ks]
    got, _ = reduce(G, buckets, c)
    want = R.g1_mul(R.G1_GEN, sum((b + 1) * k for b, k in enumerate(ks)) % R.R_MOD)
    assert R.jac_to_affine(got[0] if not got[2] else R.JAC_ID) == want, f"c = {c}: reduction differs on curve points"
