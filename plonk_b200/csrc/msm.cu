// Pippenger bucket MSM into BLS12-381 G1 on sm_90a (H100).
//
// Replaces dusk_bls12_381::multiscalar_mul::msm_variable_base as called by CommitKey::commit
// (reference src/commitment_scheme/kzg10/key.rs:376-388) plus the projective->affine step of
// Commitment::from (src/commitment_scheme/kzg10/commitment.rs:89-93).  The result of an MSM is a
// group element, canonical once normalised to affine, so the schedule is free; ours is built for
// an 80 GB HBM part whose commit key never changes during the life of a Prover:
//
//   * upload: for every base P_i the multiples 2^(c*w) * P_i (w < W = ceil(256/c)) are computed
//     once and kept in HBM as affine points.  All W windows of a scalar then feed ONE set of
//     2^(c-1) buckets (signed digits), so there is a single bucket reduction per MSM instead of
//     one per window and no doubling chain at the end.
//   * per call: (1) scalars leave Montgomery form and are recoded into signed c-bit digits; a
//     histogram of bucket sizes is built with one integer atomic per digit; (2) an exclusive scan
//     turns it into bucket offsets; (3) (point,sign) references are scattered into bucket order;
//     (4) bucket accumulation: SPLIT threads per bucket add their share of the bucket's points
//     with XYZZ mixed additions (8M + 2S each) - this is where the G1 adds of the workload are;
//     (5) bucket reduction sum_b (b+1) B_b: row and column sums of the buckets laid out 8 to a row,
//     then plain sums of the row sums split by the digits of the row index; the last few dozen
//     additions (Horner over those digits) and the single inversion for the affine result run on
//     the host.
//   * `batch` scalar vectors against the same key are processed by the same launches
//     (Prover::commit_polynomials commits 4 polynomials at once, src/compiler/prover.rs:187-210).
#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "internal.cuh"
#include "fp_inv.cuh"
#include "g1.cuh"
#include "host_field.h"

struct pb200_srs {
  size_t n_points;
  int c;  // window width in bits
  int W;  // number of windows
  uint4* table;  // [W][n_points] affine, 96 bytes each
  bool has_inf;  // some entry of the table is the identity (k_msm_digits then leaves such entries out)
};

namespace pb {

static constexpr int kGroup = 8;
// Over-long buckets leave the one-thread-group-per-bucket kernel: they are cut into chunks of kHeavyChunk
// entries, one warp per chunk, and the chunk sums are added per bucket afterwards.  "Over-long" is decided
// on the device from the MSM's actual load (k_msm_scan): more than max(kHeavyMin, kHeavyFactor x the average
// bucket) entries.  A dense MSM (uniform scalars, average 32..64) never has such a bucket; a sparse one (the
// wire VALUES of a circuit: average 2, a tail of buckets with dozens to tens of thousands of entries) sends
// its tail there, so that no lane of k_msm_accumulate walks more than a few dozen entries.
// A warp's chunk is 8 entries per lane (kHeavyChunk) when the MSM is alone on the GPU, and 32 per lane
// (kHeavyChunkWide) when other proofs keep the machine busy: the 5-level shuffle tree that ends every chunk
// costs 5 full additions per lane, 60 % extra work on 8 mixed additions and 15 % on 32.
static constexpr unsigned kHeavyMin = 32, kHeavyFactor = 4;
static constexpr unsigned kHeavyChunk = 256, kHeavyChunkWide = 1024;

PB_D G1Affine ld_affine(const uint4* p, size_t i) {
  const uint4* q = p + 6 * i;
  uint4 a0 = __ldg(q), a1 = __ldg(q + 1), a2 = __ldg(q + 2), b0 = __ldg(q + 3), b1 = __ldg(q + 4), b2 = __ldg(q + 5);
  G1Affine r;
  r.x.v[0] = a0.x; r.x.v[1] = a0.y; r.x.v[2] = a0.z; r.x.v[3] = a0.w;
  r.x.v[4] = a1.x; r.x.v[5] = a1.y; r.x.v[6] = a1.z; r.x.v[7] = a1.w;
  r.x.v[8] = a2.x; r.x.v[9] = a2.y; r.x.v[10] = a2.z; r.x.v[11] = a2.w;
  r.y.v[0] = b0.x; r.y.v[1] = b0.y; r.y.v[2] = b0.z; r.y.v[3] = b0.w;
  r.y.v[4] = b1.x; r.y.v[5] = b1.y; r.y.v[6] = b1.z; r.y.v[7] = b1.w;
  r.y.v[8] = b2.x; r.y.v[9] = b2.y; r.y.v[10] = b2.z; r.y.v[11] = b2.w;
  return r;
}
PB_D void st_fp(uint4* q, const Fp& f) {
  q[0] = make_uint4(f.v[0], f.v[1], f.v[2], f.v[3]);
  q[1] = make_uint4(f.v[4], f.v[5], f.v[6], f.v[7]);
  q[2] = make_uint4(f.v[8], f.v[9], f.v[10], f.v[11]);
}
PB_D Fp ld_fp(const uint4* q) {
  uint4 a = q[0], b = q[1], c = q[2];
  Fp f;
  f.v[0] = a.x; f.v[1] = a.y; f.v[2] = a.z; f.v[3] = a.w;
  f.v[4] = b.x; f.v[5] = b.y; f.v[6] = b.z; f.v[7] = b.w;
  f.v[8] = c.x; f.v[9] = c.y; f.v[10] = c.z; f.v[11] = c.w;
  return f;
}
PB_D void st_affine(uint4* p, size_t i, const G1Affine& a) {
  st_fp(p + 6 * i, a.x);
  st_fp(p + 6 * i + 3, a.y);
}
// Stored XYZZ points are canonical (192 bytes): the host finish and the multi-GPU combine read the limbs.
PB_D void st_xyzz(uint4* p, size_t i, const G1Xyzz& a) {
  const G1Xyzz c = a.canonical();
  st_fp(p + 12 * i, c.x.raw());
  st_fp(p + 12 * i + 3, c.y.raw());
  st_fp(p + 12 * i + 6, c.zz.raw());
  st_fp(p + 12 * i + 9, c.zzz.raw());
}
PB_D G1Xyzz ld_xyzz(const uint4* p, size_t i) {
  G1Xyzz a;
  a.x = FpR::from(ld_fp(p + 12 * i));
  a.y = FpR::from(ld_fp(p + 12 * i + 3));
  a.zz = FpR::from(ld_fp(p + 12 * i + 6));
  a.zzz = FpR::from(ld_fp(p + 12 * i + 9));
  return a;
}

// table[w][i] = 2^(c*w) * table[0][i]; *n_inf counts the points that are the identity in some window
__global__ void k_msm_precompute(uint4* table, size_t n, int c, int W, unsigned* n_inf) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p = ld_affine(table, i);
  bool inf = p.is_inf();
  for (int w = 1; w < W; w++) {
    if (!p.is_inf()) {
      G1Xyzz q = G1Xyzz::from_affine(p);
      for (int k = 0; k < c; k++) q = xyzz_dbl(q);
      p = xyzz_to_affine(q);
    }
    inf |= p.is_inf();
    st_affine(table, (size_t)w * n + i, p);
  }
  if (inf) atomicAdd(n_inf, 1u);
}

// PublicParameters::setup restated for the device (reference src/commitment_scheme/kzg10/srs.rs:61-100):
// out[i] = [g_scalar * x^i] G1::generator, normalised to affine, by fixed-base multiplication.
//
// The generator never changes, so its signed-window table is built once per process (srs_gen_table):
//   T[w][d - 1] = [d * 2^(kSetupC * w)] G,   w < kSetupW, d = 1 .. 2^(kSetupC - 1)   (32 x 128 points, 384 KiB).
// A scalar below r < 2^255 recoded into signed 8-bit digits has kSetupW = 32 windows, the top one at most 128, so
// [s]G is one mixed addition per non-zero digit and no doubling at all.
static constexpr int kSetupC = 8, kSetupW = 32, kSetupHalf = 1 << (kSetupC - 1);

PB_D G1Affine g1_generator() {  // G1Affine::generator(), Montgomery limbs
  const uint32_t gx[12] = {0xfd530c16u, 0x5cb38790u, 0x9976fff5u, 0x7817fc67u, 0x143ba1c1u, 0x154f95c7u,
                           0xf3d0e747u, 0xf0ae6acdu, 0x21dbf440u, 0xedce6eccu, 0x9e0bfb75u, 0x12017741u};
  const uint32_t gy[12] = {0x0ce72271u, 0xbaac93d5u, 0x7918fd8eu, 0x8c22631au, 0x570725ceu, 0xdd595f13u,
                           0x50405194u, 0x51ac5829u, 0xad0059c0u, 0x0e1c8c3fu, 0x5008a26au, 0x0bbc3efcu};
  G1Affine g;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    g.x.v[k] = gx[k];
    g.y.v[k] = gy[k];
  }
  return g;
}

// One thread per table entry: [d * 2^(8w)] G by double-and-add (once per process, 4096 threads).
__global__ void __launch_bounds__(128) k_srs_gen_table(uint4* table) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= kSetupW * kSetupHalf) return;
  const int w = t / kSetupHalf, d = t % kSetupHalf + 1;
  uint32_t k[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // d * 2^(8w) < 2^255
  const int bit = kSetupC * w;
  k[bit / 32] = (uint32_t)d << (bit % 32);
  if (bit % 32 > 24) k[bit / 32 + 1] = (uint32_t)d >> (32 - bit % 32);
  st_affine(table, t, xyzz_to_affine(xyzz_mul(G1Xyzz::from_affine(g1_generator()), k, 8)));
}

// Thread t owns the run [t * run, min(n, (t + 1) * run)) of powers.  It forms g_scalar * x^i by one pow for the first
// index and one Fr product per step, sums one table point per non-zero signed digit into an XYZZ accumulator, and
// normalises the whole run with one inversion (Montgomery's trick): per point it keeps X * ZZZ and Y * ZZ in out[i] and
// q = ZZ * ZZZ and the running product of the q's in `scratch` ([run][threads] pairs of Fp, so a warp's accesses are
// contiguous); then x = X ZZZ / q and y = Y ZZ / q walking the run backwards.  g_scalar * x^i is never zero - both
// draws are nonzero and r is prime - so no accumulator ends at the identity and every q is invertible.
__global__ void __launch_bounds__(128) k_srs_setup(uint4* out, size_t n, Fr x, Fr g_scalar, const uint4* __restrict__ table,
                                                   uint4* scratch, unsigned run) {
  const size_t threads = (size_t)gridDim.x * blockDim.x, t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t first = t * run;
  if (first >= n) return;
  const unsigned m = (unsigned)min((size_t)run, n - first);
  Fr p = g_scalar * x.pow_u64(first);
  Fp prod = Fp::one();
#pragma unroll 1
  for (unsigned j = 0; j < m; j++) {
    const Fr s = p.from_mont();
    p = p * x;
    G1Xyzz acc = G1Xyzz::identity();
    unsigned carry = 0;
#pragma unroll 1
    for (int w = 0; w < kSetupW; w++) {
      int d = (int)((s.v[w / 4] >> (8 * (w % 4))) & 0xffu) + (int)carry;
      carry = d > kSetupHalf;
      if (carry) d -= 1 << kSetupC;
      if (d == 0) continue;
      const G1Affine pt = ld_affine(table, (size_t)w * kSetupHalf + (d > 0 ? d : -d) - 1);
      xyzz_madd(acc, pt.x, d > 0 ? pt.y : pt.y.neg());
    }
    const Fp zz = acc.zz.canonical(), zzz = acc.zzz.canonical();
    const Fp q = zz * zzz;
    prod = prod * q;
    G1Affine xy;
    xy.x = acc.x.canonical() * zzz;
    xy.y = acc.y.canonical() * zz;
    st_affine(out, first + j, xy);
    uint4* sc = scratch + 6 * (j * threads + t);
    st_fp(sc, q);
    st_fp(sc + 3, prod);
  }
  Fp inv = fp_inv_bingcd(prod);  // 1 / (q_0 ... q_{m-1})
#pragma unroll 1
  for (unsigned j = m; j-- > 0;) {
    const uint4* sc = scratch + 6 * (j * threads + t);
    const Fp iq = j ? inv * ld_fp(sc - 6 * threads + 3) : inv;  // 1 / q_j
    inv = inv * ld_fp(sc);
    G1Affine xy;  // plain loads: out[] was written by this kernel, so not through the read-only path
    xy.x = ld_fp(out + 6 * (first + j)) * iq;
    xy.y = ld_fp(out + 6 * (first + j) + 3) * iq;
    st_affine(out, first + j, xy);
  }
}

// G1Affine::from_slice for a whole commit key (CommitKey::from_slice, reference
// src/commitment_scheme/kzg10/key.rs:319-326; PublicParameters::from_slice srs.rs:163-178): the
// 48-byte zcash encoding (big-endian x; bit 7 compressed, bit 6 infinity, bit 5 "y is the larger
// root") is decoded to the 96-byte raw layout.  One thread per point: canonical-x check, y =
// (x^3 + 4)^((p+1)/4) (p = 3 mod 4), root check, sign selection and - as G1Affine::from_bytes does -
// the prime-order subgroup check [r]P = O.  `bad` receives the smallest index of a malformed point.
__global__ void __launch_bounds__(64) k_g1_decompress(const uint8_t* in, size_t n, int check_subgroup, uint4* out, unsigned* bad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* b = in + 48 * i;
  const unsigned flags = b[0];
  Fp x;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    const int o = 44 - 4 * k;
    x.v[k] = ((uint32_t)b[o] << 24) | ((uint32_t)b[o + 1] << 16) | ((uint32_t)b[o + 2] << 8) | (uint32_t)b[o + 3];
  }
  x.v[11] &= 0x1fffffffu;
  bool ok = (flags & 0x80u) != 0;
  G1Affine pt;
  pt.x = Fp::zero();
  pt.y = Fp::zero();
  if (flags & 0x40u) {
    ok = ok && x.is_zero() && !(flags & 0x20u);
  } else {
    bool lt = false;  // x < p, compared from the top limb
#pragma unroll
    for (int k = 11; k >= 0; k--) {
      const uint32_t m = FpParams::MOD(k);
      if (x.v[k] != m) {
        lt = x.v[k] < m;
        break;
      }
    }
    ok = ok && lt;
    if (ok) {
      const Fp xm = x.to_mont();
      const Fp four = Fp::one().dbl().dbl();
      const Fp y2 = xm.sqr() * xm + four;
      uint32_t e[12];  // (p + 1) / 4
#pragma unroll
      for (int k = 0; k < 12; k++) e[k] = FpParams::MOD(k);
      e[0] += 1u;  // no carry: the low limb of p is 0xffffaaab
#pragma unroll
      for (int k = 0; k < 12; k++) e[k] = (e[k] >> 2) | (k < 11 ? e[k + 1] << 30 : 0u);
      Fp y = y2.pow(e, 12);
      ok = y.sqr() == y2;
      // y is "the larger root" iff y > p - y as integers
      const Fp yc = y.from_mont(), nc = y.neg().from_mont();
      bool larger = false;
#pragma unroll
      for (int k = 11; k >= 0; k--) {
        if (yc.v[k] != nc.v[k]) {
          larger = yc.v[k] > nc.v[k];
          break;
        }
      }
      if (larger != ((flags & 0x20u) != 0)) y = y.neg();
      pt.x = xm;
      pt.y = y;
      if (ok && check_subgroup) {
        G1Xyzz acc = G1Xyzz::identity();
#pragma unroll 1
        for (int w = 7; w >= 0; w--) {
          const uint32_t word = FrParams::MOD(w);
#pragma unroll 1
          for (int bit = 31; bit >= 0; bit--) {
            acc = xyzz_dbl(acc);
            if ((word >> bit) & 1u) xyzz_madd(acc, pt.x, pt.y);
          }
        }
        ok = acc.is_inf();
      }
    }
  }
  if (!ok) {
    atomicMin(bad, (unsigned)i);
    pt.x = Fp::zero();
    pt.y = Fp::zero();
  }
  st_affine(out, i, pt);
}

// CommitKey::from_raw_var_bytes (reference src/commitment_scheme/kzg10/key.rs:258-298) validates every
// point of a raw-encoded key with is_on_curve() & is_torsion_free(); this is that check for points already
// in the 96-byte raw layout (identity = zeros, always valid).  One thread per point; `bad` receives the
// smallest index of an invalid point.
__global__ void __launch_bounds__(64) k_g1_check_raw(const uint4* pts, size_t n, unsigned* bad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const G1Affine p = ld_affine(pts, i);
  if (p.is_inf()) return;
  const Fp four = Fp::one().dbl().dbl();
  bool ok = p.y.sqr() == p.x.sqr() * p.x + four;
  if (ok) {
    G1Xyzz acc = G1Xyzz::identity();
#pragma unroll 1
    for (int w = 7; w >= 0; w--) {
      const uint32_t word = FrParams::MOD(w);
#pragma unroll 1
      for (int bit = 31; bit >= 0; bit--) {
        acc = xyzz_dbl(acc);
        if ((word >> bit) & 1u) xyzz_madd(acc, p.x, p.y);
      }
    }
    ok = acc.is_inf();
  }
  if (!ok) atomicMin(bad, (unsigned)i);
}

// G1Affine::to_bytes for a whole commit key (CommitKey::to_var_bytes, key.rs:303-308), the inverse of
// k_g1_decompress and the device twin of pbh::g1_compress_raw: big-endian canonical x with bit 7 set, bit 5 when
// y > (p - 1) / 2; the identity is 0xc0 and zeros.  One thread per point, 48 bytes out as three 128-bit stores.
__global__ void __launch_bounds__(128) k_g1_compress(const uint4* __restrict__ pts, size_t n, uint4* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const G1Affine p = ld_affine(pts, i);
  Fp x = Fp::zero();
  uint32_t flags = 0xc0000000u;
  if (!p.is_inf()) {
    x = p.x.from_mont();
    // y is "the larger root" iff y > p - y as integers
    const Fp yc = p.y.from_mont(), nc = p.y.neg().from_mont();
    bool larger = false;
#pragma unroll
    for (int k = 11; k >= 0; k--) {
      if (yc.v[k] != nc.v[k]) {
        larger = yc.v[k] > nc.v[k];
        break;
      }
    }
    flags = 0x80000000u | (larger ? 0x20000000u : 0u);
  }
  x.v[11] |= flags;
  uint32_t be[12];  // byte 4k..4k+3 of the encoding = limb 11-k, most significant byte first
#pragma unroll
  for (int k = 0; k < 12; k++) be[k] = __byte_perm(x.v[11 - k], 0u, 0x0123);
  uint4* o = out + 3 * i;
  o[0] = make_uint4(be[0], be[1], be[2], be[3]);
  o[1] = make_uint4(be[4], be[5], be[6], be[7]);
  o[2] = make_uint4(be[8], be[9], be[10], be[11]);
}

// Signed-digit recoding + bucket histogram.  ebkt/epos are [batch][W][n].  inf_table is the key's table
// when it holds the identity (else null): a digit whose table entry is the identity adds nothing and
// gets no entry, so that the bucket walk never meets the identity.
__global__ void k_msm_digits(const uint4* scalars, size_t n, size_t stride, int c, int W, unsigned nb,
                             const uint4* inf_table, size_t n_table, size_t first, unsigned* counts, unsigned* ebkt,
                             unsigned* epos) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned b = blockIdx.y;
  const uint4* sp = scalars + 2 * ((size_t)b * stride + i);
  uint4 lo = __ldg(sp), hi = __ldg(sp + 1);
  Fr s;
  s.v[0] = lo.x; s.v[1] = lo.y; s.v[2] = lo.z; s.v[3] = lo.w;
  s.v[4] = hi.x; s.v[5] = hi.y; s.v[6] = hi.z; s.v[7] = hi.w;
  s = s.from_mont();
  const unsigned mask = (1u << c) - 1u, half = 1u << (c - 1);
  unsigned carry = 0;
  for (int w = 0; w < W; w++) {
    const int bit = w * c;
    const int word = bit >> 5, off = bit & 31;
    unsigned val = 0;
    if (word < 8) {
      val = s.v[word] >> off;
      if (off && word + 1 < 8) val |= s.v[word + 1] << (32 - off);
      val &= mask;
    }
    unsigned d = val + carry;
    unsigned sign = 0;
    if (d > half) {
      d = (1u << c) - d;
      sign = 1;
      carry = 1;
    } else {
      carry = 0;
    }
    const size_t slot = ((size_t)b * W + w) * n + i;
    if (d != 0 && inf_table && ld_affine(inf_table, (size_t)w * n_table + first + i).is_inf()) d = 0;
    if (d == 0) {
      ebkt[slot] = 0xffffffffu;
    } else {
      const unsigned bucket = d - 1;
      ebkt[slot] = (bucket << 1) | sign;
      epos[slot] = atomicAdd(&counts[(size_t)b * nb + bucket], 1u);
    }
  }
}

// Exclusive scan of counts[b][0..nb) into offsets[b][0..nb]; one CTA of 1024 threads per b.
// The same CTA also emits `order`: the bucket ids sorted by descending size (counting sort on the
// clipped size), so that the threads of a warp in k_msm_accumulate get buckets of near-equal length
// and the warp does not idle on its longest lane.
__global__ void __launch_bounds__(1024) k_msm_scan(const unsigned* counts, unsigned* offsets, unsigned* order, unsigned* n_heavy,
                                                   unsigned* heavy_pre, unsigned* max_len, unsigned nb, int size_shift,
                                                   unsigned heavy_chunk) {
  __shared__ unsigned sums[1024];
  __shared__ unsigned bins[1024];
  __shared__ unsigned s_nh, s_total, s_thr_units, s_max;
  const unsigned b = blockIdx.x, tid = threadIdx.x;
  const unsigned* cnt = counts + (size_t)b * nb;
  unsigned* off = offsets + (size_t)b * (nb + 1);
  unsigned* ord = order + (size_t)b * nb;
  const unsigned chunk = (nb + 1023) / 1024;
  const unsigned lo = tid * chunk, hi = min(nb, lo + chunk);
  unsigned s = 0, mx = 0;
  for (unsigned k = lo; k < hi; k++) {
    s += cnt[k];
    mx = max(mx, cnt[k]);
  }
  sums[tid] = s;
  bins[tid] = 0;
  if (tid == 0) s_max = 0;
  __syncthreads();
  if (mx) atomicMax(&s_max, mx);
  for (unsigned d = 1; d < 1024; d <<= 1) {
    unsigned v = (tid >= d) ? sums[tid - d] : 0;
    __syncthreads();
    sums[tid] += v;
    __syncthreads();
  }
  unsigned run = sums[tid] - s;
  for (unsigned k = lo; k < hi; k++) {
    off[k] = run;
    run += cnt[k];
  }
  if (tid == 1023) {
    off[nb] = sums[1023];
    s_total = sums[1023];
    max_len[b] = s_max;  // the scan loops above passed several barriers since the atomicMax
  }
  // counting sort of the buckets by size (in units of 2^size_shift entries, so that the average
  // bucket lands near bin 64 whatever the MSM size), largest first (bin 0 = size >= 1023 units)
  for (unsigned k = tid; k < nb; k += 1024) atomicAdd(&bins[1023u - min(cnt[k] >> size_shift, 1023u)], 1u);
  __syncthreads();
  const unsigned mine = bins[tid];
  sums[tid] = mine;
  __syncthreads();
  for (unsigned d = 1; d < 1024; d <<= 1) {
    unsigned v = (tid >= d) ? sums[tid - d] : 0;
    __syncthreads();
    sums[tid] += v;
    __syncthreads();
  }
  bins[tid] = sums[tid] - mine;  // exclusive start of each bin
  // buckets are ordered largest first, so the heavy ones are order[0 .. n_heavy)
  // heavy: more than thr_units size units, thr = max(kHeavyMin, kHeavyFactor * average) entries rounded up to units
  if (tid == 0) {
    const unsigned avg = s_total / nb;
    const unsigned thr = max(kHeavyMin, kHeavyFactor * avg);
    s_thr_units = min(1021u, (thr + (1u << size_shift) - 1u) >> size_shift);
  }
  __syncthreads();
  if (tid == 1022u - s_thr_units) {  // bins 0 .. 1022-thr hold the sizes > thr units
    n_heavy[b] = sums[tid];
    s_nh = sums[tid];
  }
  __syncthreads();
  for (unsigned k = tid; k < nb; k += 1024) {
    const unsigned pos = atomicAdd(&bins[1023u - min(cnt[k] >> size_shift, 1023u)], 1u);
    ord[pos] = k;
  }
  __syncthreads();  // ord[0 .. n_heavy) is complete (written by this CTA)
  // heavy_pre[h] = number of heavy_chunk-entry chunks of the heavy buckets before the h-th one
  const unsigned nh = s_nh;
  unsigned* hp = heavy_pre + (size_t)b * (nb + 1);
  const unsigned per = (nh + 1023u) / 1024u;
  const unsigned h_lo = min(nh, tid * per), h_hi = min(nh, h_lo + per);
  unsigned c = 0;
  for (unsigned h = h_lo; h < h_hi; h++) c += (cnt[ord[h]] + heavy_chunk - 1) / heavy_chunk;
  sums[tid] = c;
  __syncthreads();
  for (unsigned d = 1; d < 1024; d <<= 1) {
    unsigned v = (tid >= d) ? sums[tid - d] : 0;
    __syncthreads();
    sums[tid] += v;
    __syncthreads();
  }
  unsigned run2 = sums[tid] - c;
  for (unsigned h = h_lo; h < h_hi; h++) {
    hp[h] = run2;
    run2 += (cnt[ord[h]] + heavy_chunk - 1) / heavy_chunk;
  }
  if (tid == 1023) hp[nh] = sums[1023];
}

__global__ void k_msm_scatter(const unsigned* ebkt, const unsigned* epos, const unsigned* offsets, size_t n,
                              int W, unsigned nb, size_t n_table, size_t first, unsigned* sorted) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned w = blockIdx.y, b = blockIdx.z;
  const size_t slot = ((size_t)b * W + w) * n + i;
  const unsigned e = ebkt[slot];
  if (e == 0xffffffffu) return;
  const unsigned bucket = e >> 1, sign = e & 1u;
  const unsigned dst = offsets[(size_t)b * (nb + 1) + bucket] + epos[slot];
  sorted[(size_t)b * n * W + dst] = (unsigned)(((size_t)w * n_table + first + i) << 1) | sign;
}

PB_D G1Xyzz shfl_down_xyzz(const G1Xyzz& p, int delta, int width) {
  G1Xyzz r;
#pragma unroll
  for (int i = 0; i < 12; i++) {
    r.x.v[i] = __shfl_down_sync(0xffffffffu, p.x.v[i], delta, width);
    r.y.v[i] = __shfl_down_sync(0xffffffffu, p.y.v[i], delta, width);
    r.zz.v[i] = __shfl_down_sync(0xffffffffu, p.zz.v[i], delta, width);
    r.zzz.v[i] = __shfl_down_sync(0xffffffffu, p.zzz.v[i], delta, width);
  }
  return r;
}

// The rare step of a bucket walk, out of line so that its doubling stays off the walk's code path: acc is
// P, -P or the identity (after an earlier P + (-P)) for the entry e.
__device__ __noinline__ G1Xyzz bucket_step_cold(G1Xyzz acc, const uint4* table, unsigned e) {
  const G1Affine pt = ld_affine(table, e >> 1);
  xyzz_madd(acc, FpR::from(pt.x), signed_y(pt.y, e & 1u));
  return acc;
}

// The sum of the entries src[k], src[k + step], ... below hi (the identity when there is none).  An entry is
// (table index << 1 | sign); the table holds no identity (k_msm_digits leaves those entries out).  The first
// entry starts the sum, and the next entry's load is issued as soon as the current point has gone into its
// two products, into the same registers, so it is in flight during the rest of the addition.
PB_D G1Xyzz bucket_walk(const uint4* table, const unsigned* src, unsigned k, unsigned hi, unsigned step) {
  if (k >= hi) return G1Xyzz::identity();
  unsigned e = __ldg(src + k);
  G1Affine pt = ld_affine(table, e >> 1);
  G1Xyzz acc;
  acc.x = FpR::from(pt.x);
  acc.y = signed_y(pt.y, e & 1u);
  acc.zz = FpR::one();
  acc.zzz = FpR::one();
  k += step;
  if (k < hi) {
    e = __ldg(src + k);
    pt = ld_affine(table, e >> 1);
  }
  for (; k < hi; k += step) {
    const FpR u2 = FpR::from(pt.x) * acc.zz;
    const FpR s2 = signed_y(pt.y, e & 1u) * acc.zzz;
    const unsigned cur = e;
    if (k + step < hi) {
      e = __ldg(src + k + step);
      pt = ld_affine(table, e >> 1);
    }
    if (!xyzz_madd_distinct(acc, u2, s2)) acc = bucket_step_cold(acc, table, cur);
  }
  return acc;
}

// Bucket accumulation: thread = (bucket, part); the 2^log_split parts of a bucket are adjacent
// lanes and are merged with a warp-shuffle tree, so `sums` holds one XYZZ point per bucket
// ([batch][nb]).  Buckets are visited in `order` (largest first, near-equal sizes per warp).
template <int THREADS, int MIN_CTAS>
__global__ void __launch_bounds__(THREADS, MIN_CTAS) k_msm_accumulate(const uint4* table, const unsigned* sorted,
                                                               const unsigned* offsets, const unsigned* order,
                                                               const unsigned* n_heavy, unsigned nb, int log_split, size_t cap,
                                                               uint4* sums) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned split = 1u << log_split;
  const unsigned b = blockIdx.y;
  // the first n_heavy buckets of `order` are handled by k_msm_heavy_chunks
  const bool valid = t < ((size_t)nb << log_split) && (t >> log_split) >= n_heavy[b];
  const unsigned part = (unsigned)t & (split - 1);
  unsigned bucket = 0, lo = 0, hi = 0;
  if (valid) {
    bucket = order[(size_t)b * nb + (t >> log_split)];
    const unsigned* off = offsets + (size_t)b * (nb + 1);
    const unsigned start = off[bucket], end = off[bucket + 1];
    const unsigned chunk = (end - start + split - 1) >> log_split;
    lo = min(end, start + part * chunk);
    hi = min(end, lo + chunk);
  }
  G1Xyzz acc = bucket_walk(table, sorted + (size_t)b * cap, lo, hi, 1);
  for (int d = (int)split >> 1; d > 0; d >>= 1) {
    G1Xyzz o = shfl_down_xyzz(acc, d, (int)split);
    if (part + d < split) xyzz_add(acc, o);
  }
  if (valid && part == 0) st_xyzz(sums, (size_t)b * nb + bucket, acc);
}

// The sum lands in lane 0.  A lane whose partner is past the end of the warp gets its own value back from the
// shuffle; it skips the addition (a doubling, which would serialise with the other lanes' additions) because
// lane 0 never reads what it holds.
PB_D G1Xyzz warp_sum(G1Xyzz v) {
  const unsigned lane = threadIdx.x & 31;
  for (int d = 16; d > 0; d >>= 1) {
    G1Xyzz o = shfl_down_xyzz(v, d, 32);
    if (lane + d < 32) xyzz_add(v, o);
  }
  return v;
}

// Heavy buckets (skewed scalars: many equal coefficients, 0/1 vectors, the wire VALUES of a circuit, whose
// small entries pile tens of thousands of points onto digits 1, 2, 3 of the lowest window): the chunks of
// all heavy buckets form one work list, a warp per chunk of heavy_chunk entries (8 or 32 mixed additions per
// lane and a shuffle tree), so a 30 000-entry bucket is spread over 30..118 warps instead of being walked by one CTA.
// With uniformly random scalars there is no heavy bucket and the warps exit at once.
__global__ void __launch_bounds__(128) k_msm_heavy_chunks(const uint4* table, const unsigned* sorted, const unsigned* offsets,
                                                          const unsigned* order, const unsigned* n_heavy, const unsigned* heavy_pre,
                                                          unsigned nb, unsigned heavy_chunk, size_t cap, size_t part_cap,
                                                          uint4* partials) {
  const unsigned b = blockIdx.y;
  const unsigned nh = n_heavy[b];
  if (nh == 0) return;
  const unsigned* hp = heavy_pre + (size_t)b * (nb + 1);
  const unsigned total = hp[nh];
  const unsigned* src = sorted + (size_t)b * cap;
  const unsigned* off = offsets + (size_t)b * (nb + 1);
  const unsigned* ord = order + (size_t)b * nb;
  const unsigned lane = threadIdx.x & 31, warps = gridDim.x * 4;
  for (unsigned v = blockIdx.x * 4 + (threadIdx.x >> 5); v < total; v += warps) {
    unsigned lo = 0, hi = nh;  // the heavy bucket h with hp[h] <= v < hp[h + 1]
    while (hi - lo > 1) {
      const unsigned mid = (lo + hi) >> 1;
      if (hp[mid] <= v) lo = mid; else hi = mid;
    }
    const unsigned bucket = ord[lo];
    const unsigned start = off[bucket] + (v - hp[lo]) * heavy_chunk, end = min(off[bucket + 1], start + heavy_chunk);
    G1Xyzz acc = warp_sum(bucket_walk(table, src, start + lane, end, 32));
    if (lane == 0) st_xyzz(partials, (size_t)b * part_cap + v, acc);
  }
}

// ... and the chunk sums of each heavy bucket are added by one warp.
__global__ void __launch_bounds__(128) k_msm_heavy_combine(const uint4* partials, const unsigned* order, const unsigned* n_heavy,
                                                           const unsigned* heavy_pre, unsigned nb, size_t part_cap, uint4* sums) {
  const unsigned b = blockIdx.y;
  const unsigned nh = n_heavy[b];
  const unsigned* hp = heavy_pre + (size_t)b * (nb + 1);
  const unsigned lane = threadIdx.x & 31, warps = gridDim.x * 4;
  for (unsigned h = blockIdx.x * 4 + (threadIdx.x >> 5); h < nh; h += warps) {
    G1Xyzz acc = G1Xyzz::identity();
    for (unsigned v = hp[h] + lane; v < hp[h + 1]; v += 32) {
      G1Xyzz q = ld_xyzz(partials, (size_t)b * part_cap + v);
      xyzz_add(acc, q);
    }
    acc = warp_sum(acc);
    if (lane == 0) st_xyzz(sums, (size_t)b * nb + order[(size_t)b * nb + h], acc);
  }
}

// ---------------------------------------------------------------------------------------------
// Bucket accumulation by batched affine additions (opt-in: PB200_MSM_AFFINE=1; the XYZZ kernels above are the
// default, see DESIGN.md section 4).
//
// An affine addition needs lambda = (y2 - y1) / (x2 - x1): 2M + 1S once 1 / (x2 - x1) is known, against
// 8M + 2S for the inversion-free XYZZ mixed addition.  Inversions are shared with Montgomery's trick
// (3M per element), which needs MANY INDEPENDENT additions at a time - a serial walk along a bucket has
// none.  So the entries of every bucket are added as a tree: in round r the surviving elements
// (2i, 2i + 1) of each bucket are added pairwise, all pairs of all buckets being independent; a bucket of L
// entries is done after ceil(log2 L) rounds, and the total number of additions is unchanged (L - 1).
//   * Layout.  Round 0 reads table points through the sorted (point, sign) references, bucket b at
//     [off[b], off[b] + L).  The output of round r is layout r + 1: bucket b keeps ceil(L_r / 2) elements at
//     off_{r+1}[b] = (off_r[b] + b) >> 1, which never overlaps its neighbour and shrinks the buffers by half
//     per round (two ping-pong buffers of cap/2 + nb and cap/4 + nb points).  A bucket's last addition
//     writes sums[b]; single-entry buckets are copied there by round 0; sums is pre-zeroed (identity).
//   * Work split.  A thread owns kAffK consecutive input POSITIONS of the round's layout, whatever buckets
//     they belong to (binary search for the first one), i.e. up to kAffK/2 pairs: a 30 000-entry bucket and
//     30 000 single-pair buckets are the same work list.  No bucket ordering, no heavy-bucket path.
//   * A round is three launches.  k_msm_affine_fwd: the thread lists its pairs, then walks them with
//     d_i = x2 - x1 (2 y1 for a doubling, 1 when a pair needs no division: an identity operand or P + (-P)),
//     storing the running product before d_i; the CTA's 128 thread products are combined by shuffles into
//     F_t (the product of the OTHER threads) and the CTA total T_c.  k_fp_batch_inverse: all T_c of the round
//     inverted with ONE inversion - a binary extended GCD on the integer-add pipe by a single lane.
//     k_msm_affine_back: 1 / (thread product) = F_t / T_c; the thread walks back, 1 / d_i = (running inverse)
//     x (stored prefix), and finishes each addition (operands of the next pair staged by cp.async):
//     5M + 1S + ~0.4M of sharing per addition, 32 % fewer multiply instructions than XYZZ - and ~500 bytes
//     of memory traffic per pair against 96 per XYZZ addition, which is why it does not win (DESIGN.md).
// ---------------------------------------------------------------------------------------------
static constexpr int kAffK = 64;         // input positions per thread
static constexpr int kAffThreads = 128;  // 4096 pairs share one inversion

PB_D unsigned aff_off(unsigned o, unsigned b, int r) {
  for (int i = 0; i < r; i++) o = (o + b) >> 1;
  return o;
}
PB_D unsigned aff_len(unsigned L, int r) { return (L + (1u << r) - 1u) >> r; }

PB_D Fp shfl_fp(const Fp& a, int src_lane) {
  Fp r;
#pragma unroll
  for (int i = 0; i < 12; i++) r.v[i] = __shfl_sync(0xffffffffu, a.v[i], src_lane);
  return r;
}
PB_D Fp shfl_up_fp(const Fp& a, int d) {
  Fp r;
#pragma unroll
  for (int i = 0; i < 12; i++) r.v[i] = __shfl_up_sync(0xffffffffu, a.v[i], d);
  return r;
}
PB_D Fp shfl_down_fp(const Fp& a, int d) {
  Fp r;
#pragma unroll
  for (int i = 0; i < 12; i++) r.v[i] = __shfl_down_sync(0xffffffffu, a.v[i], d);
  return r;
}

// What one pair needs: the divisor and, later, the numerator of lambda.
//   kind 0: generic addition (d = x2 - x1, num = y2 - y1);  1: doubling (d = 2 y1, num = 3 x1^2);
//   2: result = P1 (P2 is the identity);  3: result = P2;  4: result = identity (P2 = -P1)
PB_D int aff_classify(const G1Affine& p1, const G1Affine& p2, Fp* d) {
  if (p2.is_inf()) return 2;
  if (p1.is_inf()) return 3;
  const Fp dx = p2.x - p1.x;
  if (!dx.is_zero()) {
    *d = dx;
    return 0;
  }
  if (p1.y == p2.y && !p1.y.is_zero()) {
    *d = p1.y.dbl();
    return 1;
  }
  return 4;
}
PB_D G1Affine aff_finish(int kind, const G1Affine& p1, const G1Affine& p2, const Fp& inv_d) {
  if (kind == 2) return p1;
  if (kind == 3) return p2;
  G1Affine r;
  if (kind == 4) {
    r.x = Fp::zero();
    r.y = Fp::zero();
    return r;
  }
  Fp num;
  if (kind == 0) {
    num = p2.y - p1.y;
  } else {
    const Fp xx = p1.x.sqr();
    num = xx.dbl() + xx;
  }
  const Fp lam = num * inv_d;
  r.x = lam.sqr() - p1.x - p2.x;
  r.y = lam * (p1.x - r.x) - p1.y;
  return r;
}

struct AffRound {
  const uint4* table;      // commit-key table (round 0 operands)
  const unsigned* sorted;  // [batch][cap] (point, sign) references in bucket order (round 0)
  const uint4* in;         // [batch][in_cap] points of layout r (r > 0)
  uint4* out;              // [batch][out_cap] layout r + 1
  const unsigned* offsets; // [batch][nb + 1]
  const unsigned* max_len; // [batch] longest bucket
  uint4* prefix;           // [batch][pair slots] running products (48 B each)
  uint4* desc;             // [batch][pair slots] (first operand, second operand, output slot, -)
  uint4* sums;             // [batch][nb] affine bucket sums
  uint4* factor;           // [batch][threads] product of the other threads of the CTA (48 B)
  uint4* ctot;             // [batch][ctas_max] CTA totals, inverted in place between the two kernels
  unsigned* npairs;        // [batch][threads]
  unsigned nb;
  size_t cap, in_cap, out_cap, slots;  // slots = threads per batch entry * kAffK / 2
  unsigned threads;                    // threads per batch entry in this round
  unsigned ctas_max;                   // stride of ctot
  int r;
};

// Operand addressing.  Round 0: an operand is a (table index << 1 | sign) reference; later rounds: a position
// in the input layout.
template <bool FIRST>
PB_D const uint4* aff_src(const AffRound& a, unsigned b, unsigned ref) {
  return FIRST ? a.table + 6 * (size_t)(ref >> 1) : a.in + 6 * ((size_t)b * a.in_cap + ref);
}
template <bool FIRST>
PB_D G1Affine aff_load(const AffRound& a, unsigned b, unsigned ref) {
  const uint4* q = aff_src<FIRST>(a, b, ref);
  G1Affine p;
  p.x = ld_fp(q);
  p.y = ld_fp(q + 3);
  if (FIRST && (ref & 1u) && !p.is_inf()) p.y = p.y.neg();
  return p;
}
PB_D void aff_store(const AffRound& a, unsigned b, unsigned slot, const G1Affine& p) {
  if (slot & 0x80000000u)
    st_affine(a.sums, (size_t)b * a.nb + (slot & 0x7fffffffu), p);
  else
    st_affine(a.out, (size_t)b * a.out_cap + slot, p);
}
PB_D void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}

// A round is three launches, so that no multiply-pipe time is spent waiting for an inversion:
//   k_msm_affine_fwd   phases A1 + A2 and the CTA's product tree: every thread leaves its pair list, the running
//                      products, its pair count and the factor F_t = (product of all OTHER threads of the CTA);
//                      the CTA leaves its total T_c.
//   k_fp_batch_inverse all T_c of the round (a few hundred) inverted together: one CTA per batch entry, serial
//                      Montgomery chains + warp scans + ONE binary-GCD inversion.
//   k_msm_affine_back  1 / (thread product) = (1 / T_c) * F_t, then phase C.
template <bool FIRST>
__global__ void __launch_bounds__(kAffThreads, 4) k_msm_affine_fwd(AffRound a) {
  __shared__ uint4 sh_tot[4][3];
  const unsigned b = blockIdx.y;
  const int r = a.r;
  if (r > 0 && (1u << r) >= a.max_len[b]) return;  // every bucket is finished (uniform per CTA)
  const unsigned* off = a.offsets + (size_t)b * (a.nb + 1);
  const unsigned nb = a.nb;
  const unsigned t = blockIdx.x * kAffThreads + threadIdx.x;
  const unsigned total = aff_off(off[nb], nb, r);  // end of layout r
  const unsigned pos0 = t * kAffK, pos1 = min(total, pos0 + kAffK);
  const size_t slot0 = (size_t)b * a.slots + t;  // pair i of this thread lives at slot0 + i * threads
  int np = 0;
  // ---- phase A1: list this thread's pairs (no point is touched yet); move the odd elements on ----
  if (pos0 < total) {
    // first bucket whose range reaches past pos0: the largest bk with off_r[bk] <= pos0
    unsigned lo = 0, hi = nb;  // off_r[0] = 0 <= pos0
    while (hi - lo > 1) {
      const unsigned mid = (lo + hi) >> 1;
      if (aff_off(off[mid], mid, r) <= pos0) lo = mid; else hi = mid;
    }
    const unsigned* refs = a.sorted + (size_t)b * a.cap;
    for (unsigned bk = lo; bk < nb; bk++) {
      const unsigned o = aff_off(off[bk], bk, r);
      if (o >= pos1) break;
      const unsigned L0 = off[bk + 1] - off[bk];
      const unsigned L = aff_len(L0, r);
      if (L == 0) continue;
      if (L == 1) {
        if (FIRST && o >= pos0) aff_store(a, b, 0x80000000u | bk, aff_load<FIRST>(a, b, __ldg(refs + o)));  // single entry: the bucket sum
        continue;
      }
      const unsigned o_next = aff_off(off[bk], bk, r + 1);
      unsigned e = o >= pos0 ? 0u : ((pos0 - o + 1u) & ~1u);  // first even element at or after pos0
      for (; e + 1 < L && o + e < pos1; e += 2) {
        const unsigned r1 = FIRST ? __ldg(refs + o + e) : o + e, r2 = FIRST ? __ldg(refs + o + e + 1) : o + e + 1;
        a.desc[slot0 + (size_t)np * a.threads] = make_uint4(r1, r2, L == 2 ? (0x80000000u | bk) : (o_next + (e >> 1)), 0u);
        np++;
      }
      if ((L & 1u) && o + L - 1 >= pos0 && o + L - 1 < pos1)  // odd element out: moves on unchanged
        aff_store(a, b, o_next + ((L - 1) >> 1), aff_load<FIRST>(a, b, FIRST ? __ldg(refs + o + L - 1) : o + L - 1));
    }
  }
  a.npairs[(size_t)b * a.threads + t] = (unsigned)np;
  // ---- phase A2: running product of the divisors; the x coordinates of the next pair are in flight ----
  Fp run = Fp::one();
  {
    Fp nx1 = Fp::zero(), nx2 = Fp::zero();
    uint4 nds = make_uint4(0, 0, 0, 0);
    if (np > 0) {
      nds = a.desc[slot0];
      nx1 = ld_fp(aff_src<FIRST>(a, b, nds.x));
      nx2 = ld_fp(aff_src<FIRST>(a, b, nds.y));
    }
#pragma unroll 1
    for (int i = 0; i < np; i++) {
      const Fp x1 = nx1, x2 = nx2;
      const uint4 ds = nds;
      if (i + 1 < np) {
        nds = a.desc[slot0 + (size_t)(i + 1) * a.threads];
        nx1 = ld_fp(aff_src<FIRST>(a, b, nds.x));
        nx2 = ld_fp(aff_src<FIRST>(a, b, nds.y));
      }
      Fp d = x2 - x1;
      if (d.is_zero() || x1.is_zero() || x2.is_zero()) {  // rare: equal abscissae or a possible identity - look at the whole points
        d = Fp::one();
        aff_classify(aff_load<FIRST>(a, b, ds.x), aff_load<FIRST>(a, b, ds.y), &d);
      }
      st_fp(a.prefix + 3 * (slot0 + (size_t)i * a.threads), run);
      run = run * d;
    }
  }
  // ---- the CTA's product tree: F_t = product of the other 127 thread products, T_c = product of all ----
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Fp incl = run, sfx = run;
#pragma unroll 1
  for (int d = 1; d < 32; d <<= 1) {
    const Fp up = shfl_up_fp(incl, d), dn = shfl_down_fp(sfx, d);
    if (lane >= d) incl = incl * up;
    if (lane + d < 32) sfx = sfx * dn;
  }
  Fp before = shfl_up_fp(incl, 1), after = shfl_down_fp(sfx, 1);  // products of the lanes below / above
  if (lane == 0) before = Fp::one();
  if (lane == 31) after = Fp::one();
  if (lane == 31) st_fp(sh_tot[warp], incl);
  __syncthreads();
  Fp others = Fp::one();  // the other three warps
#pragma unroll
  for (int w = 0; w < 4; w++)
    if (w != warp) others = others * ld_fp(sh_tot[w]);
  st_fp(a.factor + 3 * ((size_t)b * a.threads + t), (before * after) * others);
  if (threadIdx.x == 0) st_fp(a.ctot + 3 * ((size_t)b * a.ctas_max + blockIdx.x), others * ld_fp(sh_tot[0]));
}

// In-place inverses of n Fp values per batch entry (none of them zero), one CTA of 256 threads per batch entry.
__global__ void __launch_bounds__(256) k_fp_batch_inverse(uint4* vals, uint4* scratch, unsigned n, size_t stride, const unsigned* max_len, int r) {
  __shared__ uint4 sh_tot[8][3];
  __shared__ uint4 sh_inv[8][3];
  const unsigned b = blockIdx.x;
  if (r > 0 && (1u << r) >= max_len[b]) return;
  uint4* v = vals + 3 * (size_t)b * stride;
  uint4* pre = scratch + 3 * (size_t)b * stride;
  const unsigned m = (n + 255u) / 256u, lo = min(n, threadIdx.x * m), hi = min(n, lo + m);
  Fp run = Fp::one();
  for (unsigned i = lo; i < hi; i++) {
    st_fp(pre + 3 * i, run);
    run = run * ld_fp(v + 3 * i);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Fp incl = run, sfx = run;
#pragma unroll 1
  for (int d = 1; d < 32; d <<= 1) {
    const Fp up = shfl_up_fp(incl, d), dn = shfl_down_fp(sfx, d);
    if (lane >= d) incl = incl * up;
    if (lane + d < 32) sfx = sfx * dn;
  }
  Fp before = shfl_up_fp(incl, 1), after = shfl_down_fp(sfx, 1);
  if (lane == 0) before = Fp::one();
  if (lane == 31) after = Fp::one();
  if (lane == 31) st_fp(sh_tot[warp], incl);
  __syncthreads();
  if (threadIdx.x == 0) {
    Fp w[8], pf[8];
    Fp acc = Fp::one();
    for (int k = 0; k < 8; k++) {
      w[k] = ld_fp(sh_tot[k]);
      pf[k] = acc;
      acc = acc * w[k];
    }
    Fp inv = fp_inv_bingcd(acc);
    for (int k = 7; k >= 0; k--) {
      st_fp(sh_inv[k], inv * pf[k]);  // 1 / w[k]
      inv = inv * w[k];
    }
  }
  __syncthreads();
  Fp inv_run = ld_fp(sh_inv[warp]) * (before * after);  // 1 / (this thread's product)
  for (unsigned i = hi; i-- > lo;) {
    const Fp x = ld_fp(v + 3 * i);
    st_fp(v + 3 * i, inv_run * ld_fp(pre + 3 * i));
    inv_run = inv_run * x;
  }
}

template <bool FIRST>
__global__ void __launch_bounds__(kAffThreads, 4) k_msm_affine_back(AffRound a) {
  extern __shared__ __align__(16) uint4 sh_stage[];  // [kAffThreads][15]: the next pair's operands and running product
  const unsigned b = blockIdx.y;
  if (a.r > 0 && (1u << a.r) >= a.max_len[b]) return;
  const unsigned t = blockIdx.x * kAffThreads + threadIdx.x;
  const size_t slot0 = (size_t)b * a.slots + t;
  const int np = (int)a.npairs[(size_t)b * a.threads + t];
  if (np == 0) return;
  uint4* stage = sh_stage + 15 * threadIdx.x;
  auto fetch = [&](int i) {
    const size_t s = slot0 + (size_t)i * a.threads;
    const uint4 ds = a.desc[s];
    const uint4 *q1 = aff_src<FIRST>(a, b, ds.x), *q2 = aff_src<FIRST>(a, b, ds.y), *q3 = a.prefix + 3 * s;
#pragma unroll
    for (int k = 0; k < 6; k++) {
      cp_async16(stage + k, q1 + k);
      cp_async16(stage + 6 + k, q2 + k);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) cp_async16(stage + 12 + k, q3 + k);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  fetch(np - 1);
  // 1 / (this thread's product) = (1 / T_c) * F_t
  Fp inv_run = ld_fp(a.ctot + 3 * ((size_t)b * a.ctas_max + blockIdx.x)) * ld_fp(a.factor + 3 * ((size_t)b * a.threads + t));
  // ---- phase C: walk back, finish the additions; pair i - 1 is fetched while pair i is computed ----
#pragma unroll 1
  for (int i = np - 1; i >= 0; i--) {
    const uint4 ds = a.desc[slot0 + (size_t)i * a.threads];
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    G1Affine p1, p2;
    p1.x = ld_fp(stage); p1.y = ld_fp(stage + 3);
    p2.x = ld_fp(stage + 6); p2.y = ld_fp(stage + 9);
    const Fp pre = ld_fp(stage + 12);
    if (i > 0) fetch(i - 1);  // the slot has been read: reuse it
    if (FIRST) {
      if ((ds.x & 1u) && !p1.is_inf()) p1.y = p1.y.neg();
      if ((ds.y & 1u) && !p2.is_inf()) p2.y = p2.y.neg();
    }
    Fp d = Fp::one();
    const int kind = aff_classify(p1, p2, &d);
    const Fp inv_d = inv_run * pre;
    inv_run = inv_run * d;
    aff_store(a, b, ds.z, aff_finish(kind, p1, p2, inv_d));
  }
}

// ---------------------------------------------------------------------------------------------
// Bucket reduction  R = sum_b (b + 1) B_b.  A lone warp needs ~10 us per dependent full addition (a dozen
// carry-chained Fp products), and a reduction launch holds its registers for as long as its longest thread
// runs, so the reduction is built wide and shallow at about the work of the old running-sum scheme.  Write
// the bucket index as b = g G + j (g = kGroup buckets per row G, column j < g):
//        R = sum_j (j + 1) T_j + g sum_G G S_G,   T_j = sum_G B[gG + j],   S_G = sum_j B[gG + j]
//   A. k_msm_rows_cols: one thread per row sums its g buckets (S_G); one thread per run of kColRun rows of
//      one column sums that piece of the column (partial T_j).  g - 1 = 7 serial additions per thread.
//   B. k_msm_lists: the group index G is cut into digits of <= 4 bits; class (j, v) is the plain sum of S_G
//      over the groups whose digit j equals v; column list j is the sum of the partials of column j.  One
//      warp per (list, chunk of kListChunk members): 8 serial additions per lane + a 5-level shuffle tree.
//      Lists of more than kFinalChunks chunks (windows of 20 bits) have their chunk sums added by one more
//      warp tree per list (k_msm_fold).
//   C. k_msm_final: one warp per digit turns its 16 class sums into D_j = sum_v v C_{j,v} (suffix scan +
//      reduce); one more warp turns the g column sums into sum_j (j + 1) T_j the same way.  The host finishes
//      with a Horner over the digits (a dozen doublings, ~10 us) and the affine normalisation.
// For c = 16: 2^12 rows, 2^12 column partials, 48 classes of 256 members, 8 columns of 512 partials - about
// 2.25 * 2^15 full additions, at most 7 + (7 + 5) + (1 + 4 + 4) = 28 of them dependent (38 for the running-sum
// scheme it replaces), over 8192 threads per MSM in the widest launch (4096 before).
// ---------------------------------------------------------------------------------------------
static constexpr unsigned kColRun = 8;        // rows per partial column sum
static constexpr unsigned kListChunk = 256;   // members of a list summed by one warp
static constexpr unsigned kFinalChunks = 4;   // chunk sums per list that k_msm_final adds serially

struct DigitPlan {
  int ndig;
  int shift[8];
  int bits[8];
  int first_class[8];  // prefix sum of 2^bits
  int n_digit_classes;
  int n_columns;       // g: column lists after the digit classes
  int nlists;
};

template <bool AFFINE>
PB_D void add_bucket(G1Xyzz& acc, const uint4* sums, size_t i) {
  if (AFFINE) {  // bucket sums left by the batched-affine rounds: a mixed addition
    const G1Affine q = ld_affine(sums, i);
    if (!q.is_inf()) xyzz_madd(acc, q.x, q.y);
  } else {
    xyzz_add(acc, ld_xyzz(sums, i));
  }
}

// Threads [0, n_groups) of a batch entry: row sums S ([batch][n_groups]); threads [n_groups, n_groups + nb / col_run):
// partial column sums P ([batch][g][n_groups / col_run]).
template <bool AFFINE>
__global__ void __launch_bounds__(64) k_msm_rows_cols(const uint4* sums, unsigned nb, unsigned g, unsigned col_run, uint4* S, uint4* P) {
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned n_groups = nb / g, n_parts = n_groups / col_run;
  const unsigned b = blockIdx.y;
  const size_t base = (size_t)b * nb;
  G1Xyzz acc = G1Xyzz::identity();
  if (t < n_groups) {
    for (unsigned j = 0; j < g; j++) add_bucket<AFFINE>(acc, sums, base + (size_t)t * g + j);
    st_xyzz(S, (size_t)b * n_groups + t, acc);
  } else if (t < n_groups + g * n_parts) {
    const unsigned u = t - n_groups, j = u / n_parts, part = u % n_parts;
    for (unsigned k = 0; k < col_run; k++) add_bucket<AFFINE>(acc, sums, base + (size_t)(part * col_run + k) * g + j);
    st_xyzz(P, ((size_t)b * g + j) * n_parts + part, acc);
  }
}

// One warp per (list, chunk of kListChunk members); 4 warps per CTA.  out is [batch][nlists][chunks].
__global__ void __launch_bounds__(128) k_msm_lists(const uint4* S, const uint4* P, unsigned n_groups, unsigned n_parts,
                                                   DigitPlan plan, unsigned chunks, uint4* out) {
  const int list = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const unsigned b = blockIdx.y, chunk = blockIdx.z;
  if (list >= plan.nlists) return;
  G1Xyzz acc = G1Xyzz::identity();
  if (list < plan.n_digit_classes) {
    int j = 0;
    while (j + 1 < plan.ndig && list >= plan.first_class[j + 1]) j++;
    const unsigned v = list - plan.first_class[j];
    const int sh_j = plan.shift[j], bits_j = plan.bits[j];
    const unsigned count = n_groups >> bits_j;
    for (unsigned idx = chunk * kListChunk + lane; idx < min(count, (chunk + 1) * kListChunk); idx += 32) {
      const unsigned G = ((idx >> sh_j) << (sh_j + bits_j)) | (v << sh_j) | (idx & ((1u << sh_j) - 1u));
      xyzz_add(acc, ld_xyzz(S, (size_t)b * n_groups + G));
    }
  } else {
    const size_t col = (size_t)b * plan.n_columns + (list - plan.n_digit_classes);
    for (unsigned idx = chunk * kListChunk + lane; idx < min(n_parts, (chunk + 1) * kListChunk); idx += 32)
      xyzz_add(acc, ld_xyzz(P, col * n_parts + idx));
  }
  acc = warp_sum(acc);
  if (lane == 0) st_xyzz(out, ((size_t)b * plan.nlists + list) * chunks + chunk, acc);
}

// n_sets sets of `chunks` consecutive points -> one sum per set; one warp per set, 4 per CTA.
__global__ void __launch_bounds__(128) k_msm_fold(const uint4* in, unsigned n_sets, unsigned chunks, uint4* out) {
  const unsigned set = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (set >= n_sets) return;
  G1Xyzz acc = G1Xyzz::identity();
  for (unsigned k = lane; k < chunks; k += 32) xyzz_add(acc, ld_xyzz(in, (size_t)set * chunks + k));
  acc = warp_sum(acc);
  if (lane == 0) st_xyzz(out, set, acc);
}

// sum_{k >= first} (k + 1 - first) x_k over lanes k < n of a warp (n <= 32, a power of two): inclusive suffix
// scan, then the sum of lanes first .. n-1.  The result is in lane 0.
PB_D G1Xyzz weighted_lane_sum(G1Xyzz x, int lane, int n, int first) {
  for (int d = 1; d < n; d <<= 1) {
    G1Xyzz o = shfl_down_xyzz(x, d, 32);
    if (lane + d < n) xyzz_add(x, o);
  }
  G1Xyzz y = (lane >= first && lane < n) ? x : G1Xyzz::identity();
  for (int d = n >> 1; d > 0; d >>= 1) {
    G1Xyzz o = shfl_down_xyzz(y, d, 32);
    if (lane + d < n) xyzz_add(y, o);
  }
  return y;
}

// out is [batch][ndig + 1]: D_0 .. D_{ndig-1}, then sum_j (j + 1) T_j.
__global__ void __launch_bounds__(256) k_msm_final(const uint4* lists, DigitPlan plan, unsigned chunks, uint4* out) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned b = blockIdx.x;
  if (w >= plan.ndig && w != 7) return;
  const bool digit = w < plan.ndig;
  const int n = digit ? 1 << plan.bits[w] : plan.n_columns;
  const int first_list = digit ? plan.first_class[w] : plan.n_digit_classes;
  G1Xyzz x = G1Xyzz::identity();
  if (lane < n)
    for (unsigned ch = 0; ch < chunks; ch++) xyzz_add(x, ld_xyzz(lists, ((size_t)b * plan.nlists + first_list + lane) * chunks + ch));
  // D_j = sum_v v C_{j,v} (lane 0 holds class v = 0, weight 0); the columns carry weights 1 .. g
  const G1Xyzz y = weighted_lane_sum(x, lane, n, digit ? 1 : 0);
  if (lane == 0) st_xyzz(out, (size_t)b * (plan.ndig + 1) + (digit ? w : plan.ndig), y);
}

__global__ void k_selftest_fr_mul(const uint4* a, const uint4* b, uint4* o, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr x, y;
  uint4 t0 = a[2 * i], t1 = a[2 * i + 1];
  x.v[0] = t0.x; x.v[1] = t0.y; x.v[2] = t0.z; x.v[3] = t0.w; x.v[4] = t1.x; x.v[5] = t1.y; x.v[6] = t1.z; x.v[7] = t1.w;
  t0 = b[2 * i]; t1 = b[2 * i + 1];
  y.v[0] = t0.x; y.v[1] = t0.y; y.v[2] = t0.z; y.v[3] = t0.w; y.v[4] = t1.x; y.v[5] = t1.y; y.v[6] = t1.z; y.v[7] = t1.w;
  Fr r = x * y;
  o[2 * i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  o[2 * i + 1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
__global__ void k_selftest_fp_mul(const uint4* a, const uint4* b, uint4* o, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fp x = ld_fp(a + 3 * i), y = ld_fp(b + 3 * i);
  st_fp(o + 3 * i, x * y);
}

__global__ void k_selftest_fp_ops(const uint4* a, const uint4* b, const uint4* c, const uint4* d, uint4* o, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fp x = ld_fp(a + 3 * i), y = ld_fp(b + 3 * i), z = ld_fp(c + 3 * i), w = ld_fp(d + 3 * i);
  st_fp(o + 3 * i, x * y);
  st_fp(o + 3 * (n + i), x.sqr());
  st_fp(o + 3 * (2 * n + i), Fp::mul_sub(x, y, z, w));
}

// Register-only IMAD.WIDE throughput probe: 8 independent 64-bit accumulators per thread.
__global__ void k_imad_peak(unsigned* out, int iters, unsigned seed) {
  unsigned a = threadIdx.x * 2654435761u + seed, b = blockIdx.x * 40503u + 12345u;
  unsigned long long acc[8];
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = (unsigned long long)(a + i) << 7;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int r = 0; r < 8; r++) {
#pragma unroll
      for (int i = 0; i < 8; i++)
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"(a), "r"(b));
      a += 0x9e3779b9u;
    }
  }
  unsigned long long x = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) x ^= acc[i];
  if (x == 0x1234567ull) out[0] = (unsigned)x;  // never true in practice: keeps the chain alive
}

// Throughput probe of the carry-chained Fp product itself: every thread runs a dependent chain of
// products (x <- x * y), 1024 threads per SM-slot, so the multiply pipe is saturated by independent
// chains of different warps exactly as in the bucket kernels.  Gives the ceiling the G1 kernels are
// measured against (Fp products per second).
__global__ void __launch_bounds__(256) k_fp_product_peak(uint4* out, int iters, unsigned seed) {
  Fp x = Fp::one(), y = Fp::r2();
  x.v[0] ^= (threadIdx.x * 2654435761u + seed) & 0xffffu;  // still < p: only low bits change
  y.v[1] ^= (blockIdx.x * 40503u) & 0xffffu;
#pragma unroll 1
  for (int i = 0; i < iters; i++) {
    x = x * y;
    y = y * x;
  }
  if (x.is_zero() && y.is_zero()) st_fp(out, x);  // never true: keeps the chain alive
}

// ---------------------------------------------------------------------------------------------
// Optional in-library timing of the dominant kernel (bucket accumulation) with CUDA events on the
// launching stream; read by bench.py for the roofline line.
std::atomic<int> g_prof_on{0};
std::atomic<uint64_t> g_prof_acc_ns{0}, g_prof_acc_adds{0}, g_prof_acc_launches{0}, g_prof_acc_points{0};
// the same for sparse MSMs (fewer than a quarter of the window digits non-zero: the wire-value commitments)
std::atomic<uint64_t> g_prof_sp_ns{0}, g_prof_sp_adds{0}, g_prof_sp_launches{0}, g_prof_sp_points{0};

static int pick_window(size_t n_points) {
  if (const char* env = getenv("PB200_MSM_C")) {
    int c = atoi(env);
    if (c >= 2 && c <= 20) return c;
  }
  int lg = 0;
  while (((size_t)1 << (lg + 1)) <= n_points) lg++;
  // up to 2^16 points: c = log2(n) (~32 entries per bucket with W = 256/c windows).  Above that
  // c = 16 up to 2^19 points and c = 20 from 2^20 (tools/msm_sweep.py times the window widths).
  if (lg <= 16) return std::max(4, lg);
  return lg <= 19 ? 16 : 20;
}

static void xyzz_dev_to_host(const uint32_t* w, pbh::HXyzz* o) {
  memcpy(o->x.v, w, 48);
  memcpy(o->y.v, w + 12, 48);
  memcpy(o->zz.v, w + 24, 48);
  memcpy(o->zzz.v, w + 36, 48);
}

// What the host needs to finish an MSM whose kernels have been enqueued: the digit plan of the bucket
// reduction.  It depends on the window width of the key only, never on the number of scalars, so the
// ranks of a point-sharded MSM (pb200_msm_g1_allgather*) share it as long as their slices use the same c.
struct MsmTail {
  DigitPlan plan;
  int log_g = 0;
  int c = 0;
  uint32_t batch = 0;
  size_t words_per_entry() const { return (size_t)(plan.ndig + 1) * 48; }  // 32-bit words of one batch entry
};

// PB200_MSM_AFFINE=1: bucket accumulation by batched affine additions (k_msm_affine_fwd / _back) instead of XYZZ
static bool msm_affine_enabled() {
  static const bool on = [] {
    const char* e = getenv("PB200_MSM_AFFINE");
    return e && atoi(e) != 0;
  }();
  return on;
}

// pair slots (running product + descriptor) per batch entry: the widest round's thread count x kAffK / 2
static size_t aff_slots(size_t cap, size_t nb) {
  size_t widest = 0;
  for (int r = 0; ((size_t)1 << r) < cap || r == 0; r++) {
    const size_t positions = r == 0 ? cap : (cap >> r) + nb + 1;
    const size_t ctas = ((positions + kAffK - 1) / kAffK + kAffThreads - 1) / kAffThreads;
    widest = std::max(widest, ctas * kAffThreads);
  }
  return widest * (kAffK / 2);
}

static int msm_plan(int c, uint32_t batch, MsmTail* tail) {
  const unsigned nb = 1u << (c - 1);
  const int g = std::min<unsigned>(kGroup, nb);
  const unsigned n_groups = nb / g;
  int log_g = 0;
  while ((1 << log_g) < g) log_g++;
  DigitPlan& plan = tail->plan;
  int total_bits = 0;
  while ((1u << total_bits) < n_groups) total_bits++;
  plan.ndig = (total_bits + 3) / 4;
  if (plan.ndig > 7) return fail(PB200_ERR_INVALID_ARG, "window too wide for the bucket reduction");
  int sh = 0, cls = 0;
  for (int j = 0; j < plan.ndig; j++) {
    const int bits = (total_bits - sh) / (plan.ndig - j);  // spread evenly, low digits first
    plan.shift[j] = sh;
    plan.bits[j] = bits;
    plan.first_class[j] = cls;
    sh += bits;
    cls += 1 << bits;
  }
  plan.n_digit_classes = cls;
  plan.n_columns = g;
  plan.nlists = plan.n_digit_classes + plan.n_columns;
  tail->log_g = log_g;
  tail->c = c;
  tail->batch = batch;
  return 0;
}

// kListChunk-member chunks of the longest list of k_msm_lists (n_parts partials per column)
static unsigned reduction_chunks(const DigitPlan& plan, unsigned n_groups, unsigned n_parts) {
  unsigned chunks = (n_parts + kListChunk - 1) / kListChunk;
  for (int j = 0; j < plan.ndig; j++) chunks = std::max(chunks, ((n_groups >> plan.bits[j]) + kListChunk - 1) / kListChunk);
  return std::max(chunks, 1u);
}

// The scratch buffers of msm_enqueue in carving order; the kAff* ones exist under PB200_MSM_AFFINE=1 only.
enum MsmBuf { kResult, kCounts, kOffsets, kOrder, kMaxLen, kNHeavy, kHeavyPre, kEbkt, kEpos, kSorted, kSums, kLists, kS, kP,
              kPartials, kAffA, kAffB, kAffPre, kAffDesc, kAffFactor, kAffNpairs, kAffCtot, kAffCpre, kMsmBufs };

// What `batch` MSMs of n scalars against a key of window c (W windows) are sized from: the reduction plan, the extents
// the kernels take and the bytes of every buffer.  msm_enqueue carves exactly `bytes`; msm_workspace_bytes adds them up.
struct MsmScratch {
  MsmTail tail;
  unsigned n_groups = 0, col_run = 0, n_parts = 0, chunks = 0, ctas_max = 0;
  int g = 0;
  size_t part_cap = 0, cap_a = 0, cap_b = 0, slots = 0;
  size_t bytes[kMsmBufs] = {};
};
static int msm_scratch(int c, int W, size_t n, uint32_t batch, bool affine, MsmScratch* s) {
  PB_TRY(msm_plan(c, batch, &s->tail));
  const DigitPlan& plan = s->tail.plan;
  const size_t nb = (size_t)1 << (c - 1), cap = n * (size_t)W, B = batch;
  s->g = 1 << s->tail.log_g;  // buckets per row of the reduction
  s->n_groups = (unsigned)(nb >> s->tail.log_g);
  s->col_run = std::min(kColRun, s->n_groups);
  s->n_parts = s->n_groups / s->col_run;
  s->chunks = reduction_chunks(plan, s->n_groups, s->n_parts);
  // chunk sums of the heavy buckets: at most cap / kHeavyChunk full chunks (the narrower chunk bounds both shapes)
  // plus one ragged chunk per heavy bucket
  s->part_cap = cap / kHeavyChunk + std::min<size_t>(nb, cap / kHeavyMin) + 2;
  size_t* b = s->bytes;
  b[kResult] = B * (plan.ndig + 1) * 192;
  b[kCounts] = b[kOrder] = B * nb * 4;
  b[kOffsets] = b[kHeavyPre] = B * (nb + 1) * 4;
  b[kMaxLen] = b[kNHeavy] = B * 4;
  b[kEbkt] = b[kEpos] = b[kSorted] = B * cap * 4;
  b[kSums] = B * nb * 192;
  b[kLists] = B * plan.nlists * s->chunks * 192;
  b[kS] = B * s->n_groups * 192;
  b[kP] = B * s->g * s->n_parts * 192;
  b[kPartials] = B * s->part_cap * 192;
  if (affine) {  // two point buffers for the pairwise rounds, running products and pair descriptors, CTA totals
    s->cap_a = cap / 2 + nb + 2;
    s->cap_b = cap / 4 + nb + 2;
    s->slots = aff_slots(cap, nb);
    const size_t threads_max = s->slots / (kAffK / 2);
    s->ctas_max = (unsigned)(threads_max / kAffThreads);
    b[kAffA] = B * s->cap_a * 96;
    b[kAffB] = B * s->cap_b * 96;
    b[kAffPre] = B * s->slots * 48;
    b[kAffDesc] = B * s->slots * 16;
    b[kAffFactor] = B * threads_max * 48;
    b[kAffNpairs] = B * threads_max * 4;
    b[kAffCtot] = b[kAffCpre] = B * s->ctas_max * 48;
  }
  return 0;
}

// Enqueues every kernel of `batch` MSMs over the points [first, first + n) of the key on `st`.  The
// digit sums land in *d_result ([batch][ndig + 1] XYZZ points, carved from `scope`, so they live until
// the scope is released); nothing is synchronised.  n == 0 yields identities.
static int msm_enqueue(const pb200_srs* srs, size_t first, const uint64_t* d_scalars, size_t n, uint32_t batch, size_t stride,
                       MsmShape shape, cudaStream_t st, ScratchScope& scope, uint4** d_result, MsmTail* tail, cudaEvent_t* prof_ev,
                       const unsigned** d_totals) {
  if (first + n > srs->n_points) return fail(PB200_ERR_DEGREE_TOO_LARGE, "more scalars than commit-key points");
  const int c = srs->c, W = srs->W;
  const unsigned nb = 1u << (c - 1);
  const size_t cap = n * (size_t)W;
  if (((srs->n_points * (size_t)W) << 1) >= ((size_t)1 << 32)) return fail(PB200_ERR_INVALID_ARG, "commit key too large for 32-bit point references");
  const bool affine = msm_affine_enabled();
  MsmScratch s;
  PB_TRY(msm_scratch(c, W, n, batch, affine, &s));
  *tail = s.tail;
  const DigitPlan& plan = tail->plan;
  const unsigned n_groups = s.n_groups, col_run = s.col_run, n_parts = s.n_parts, chunks = s.chunks;
  const int g = s.g;
  uint4* result = nullptr;
  PB_ALLOC(scope, result, s.bytes[kResult]);
  *d_result = result;
  if (n == 0) {
    PB_CUDA(cudaMemsetAsync(result, 0, s.bytes[kResult], st));
    return 0;
  }

  // threads per bucket: enough CTAs to fill the machine, but at least ~8 points per thread.  Splitting a bucket
  // over 2^k lanes costs k full additions per bucket for the merge (+39 % work at k = 2 with 32 entries per
  // bucket): it buys latency when the launch is alone on the GPU and only costs throughput when other proofs
  // keep the machine busy - the caller says which (shape.split_buckets).
  int log_split = 0;
  if (shape.split_buckets) {
    const size_t avg = cap / nb;
    while (log_split < 5 && ((size_t)nb * batch << log_split) < (1u << 17) && (avg >> (log_split + 1)) >= 8) log_split++;
  }
  if (const char* env = getenv("PB200_MSM_LOG_SPLIT")) log_split = atoi(env);

  void* buf[kMsmBufs] = {};
  for (int i = kCounts; i < (affine ? kMsmBufs : kAffA); i++) PB_ALLOC(scope, buf[i], s.bytes[i]);
  unsigned *counts = (unsigned*)buf[kCounts], *offsets = (unsigned*)buf[kOffsets], *order = (unsigned*)buf[kOrder],
           *max_len = (unsigned*)buf[kMaxLen], *n_heavy = (unsigned*)buf[kNHeavy], *heavy_pre = (unsigned*)buf[kHeavyPre],
           *ebkt = (unsigned*)buf[kEbkt], *epos = (unsigned*)buf[kEpos], *sorted = (unsigned*)buf[kSorted];
  uint4 *sums = (uint4*)buf[kSums], *lists = (uint4*)buf[kLists], *S = (uint4*)buf[kS], *P = (uint4*)buf[kP],
        *partials = (uint4*)buf[kPartials];
  PB_CUDA(cudaMemsetAsync(counts, 0, s.bytes[kCounts], st));

  PB_LAUNCH(k_msm_digits, dim3(div_up(n, 128), batch), 128, 0, st, (const uint4*)d_scalars, n, stride, c, W, nb,
            srs->has_inf ? (const uint4*)srs->table : nullptr, srs->n_points, first, counts, ebkt, epos);
  int size_shift = 0;  // size unit: average bucket ~ 64 units
  while (((cap / nb) >> size_shift) > 64) size_shift++;
  const unsigned heavy_chunk = shape.wide_heavy_chunks ? kHeavyChunkWide : kHeavyChunk;
  const size_t part_cap = s.part_cap;
  PB_LAUNCH(k_msm_scan, batch, 1024, 0, st, counts, offsets, order, n_heavy, heavy_pre, max_len, nb, size_shift, heavy_chunk);
  PB_LAUNCH(k_msm_scatter, dim3(div_up(n, 256), W, batch), 256, 0, st, ebkt, epos, offsets, n, W, nb,
            srs->n_points, first, sorted);
  if (prof_ev) PB_CUDA(cudaEventRecord(prof_ev[0], st));
  if (affine) {
    // batched-affine pairwise rounds (see k_msm_affine_fwd)
    const size_t capA = s.cap_a, capB = s.cap_b, slots = s.slots;
    const unsigned ctas_max = s.ctas_max;
    int rounds = 0;
    while (((size_t)1 << rounds) < cap) rounds++;  // a bucket can hold every entry (equal scalars with equal digits)
    // input positions of round r: layout 0 is exact, layout r >= 1 has at most one slot of slack per bucket
    auto positions = [&](int r) { return r == 0 ? cap : (cap >> r) + nb + 1; };
    uint4 *bufA = (uint4*)buf[kAffA], *bufB = (uint4*)buf[kAffB], *pre = (uint4*)buf[kAffPre], *desc = (uint4*)buf[kAffDesc],
          *factor = (uint4*)buf[kAffFactor], *ctot = (uint4*)buf[kAffCtot], *cpre = (uint4*)buf[kAffCpre];
    unsigned* npairs = (unsigned*)buf[kAffNpairs];
    PB_CUDA(cudaMemsetAsync(sums, 0, (size_t)batch * nb * 96, st));
    for (int r = 0; r < rounds; r++) {
      AffRound a;
      a.table = srs->table; a.sorted = sorted; a.offsets = offsets; a.max_len = max_len; a.prefix = pre; a.desc = desc; a.sums = sums;
      a.factor = factor; a.ctot = ctot; a.npairs = npairs; a.ctas_max = ctas_max;
      a.nb = nb; a.cap = cap; a.r = r;
      a.in = (r & 1) ? bufA : bufB;   // layout r: odd layouts live in A, even ones (>= 2) in B
      a.out = (r & 1) ? bufB : bufA;  // layout r + 1
      a.in_cap = (r & 1) ? capA : capB;
      a.out_cap = (r & 1) ? capB : capA;
      const unsigned ctas = div_up(div_up(positions(r), kAffK), kAffThreads);
      a.threads = ctas * kAffThreads;
      a.slots = slots;
      const size_t stage_bytes = (size_t)kAffThreads * 15 * 16;  // one 240-byte staging slot per thread
      if (r == 0)
        PB_LAUNCH(k_msm_affine_fwd<true>, dim3(ctas, batch), kAffThreads, 0, st, a);
      else
        PB_LAUNCH(k_msm_affine_fwd<false>, dim3(ctas, batch), kAffThreads, 0, st, a);
      PB_LAUNCH(k_fp_batch_inverse, batch, 256, 0, st, ctot, cpre, ctas, (size_t)ctas_max, (const unsigned*)max_len, r);
      if (r == 0)
        PB_LAUNCH(k_msm_affine_back<true>, dim3(ctas, batch), kAffThreads, stage_bytes, st, a);
      else
        PB_LAUNCH(k_msm_affine_back<false>, dim3(ctas, batch), kAffThreads, stage_bytes, st, a);
    }
    if (prof_ev) PB_CUDA(cudaEventRecord(prof_ev[1], st));
    if (d_totals) *d_totals = offsets + nb;
    PB_LAUNCH(k_msm_rows_cols<true>, dim3(div_up(n_groups + g * n_parts, 64), batch), 64, 0, st, (const uint4*)sums, nb, (unsigned)g, col_run, S, P);
  } else {
  {
    // CTA shape: 64 threads x 4 CTAs/SM and 128 x 2 hold the same 8 warps per SM (register-limited);
    // the smaller CTA balances the tail of the launch better when there are few waves.  Forcing 12 or
    // 16 warps per SM (__launch_bounds__(128, 3 | 4)) costs 168 / 128 registers and spills.
    static const int acc_block = [] {
      const char* e = getenv("PB200_ACC_BLOCK");
      return e ? atoi(e) : 128;
    }();
    if (acc_block == 64) {
      const dim3 grid(div_up((size_t)nb << log_split, 64), batch);
      PB_LAUNCH((k_msm_accumulate<64, 4>), grid, 64, 0, st, srs->table, sorted, offsets, order, n_heavy, nb, log_split, cap, sums);
    } else {
      const dim3 grid(div_up((size_t)nb << log_split, 128), batch);
      PB_LAUNCH((k_msm_accumulate<128, 2>), grid, 128, 0, st, srs->table, sorted, offsets, order, n_heavy, nb, log_split, cap, sums);
    }
  }
  if (d_totals) *d_totals = offsets + nb;  // offsets[b][nb] = the entries of batch b (stride nb + 1)
  PB_LAUNCH(k_msm_heavy_chunks, dim3(4 * num_sms(), batch), 128, 0, st, srs->table, sorted, offsets, order, n_heavy, heavy_pre, nb, heavy_chunk, cap,
            part_cap, partials);
  PB_LAUNCH(k_msm_heavy_combine, dim3(64, batch), 128, 0, st, (const uint4*)partials, order, n_heavy, heavy_pre, nb, part_cap, sums);
  if (prof_ev) PB_CUDA(cudaEventRecord(prof_ev[1], st));  // the bucket-accumulation phase: every entry has been added once
    PB_LAUNCH(k_msm_rows_cols<false>, dim3(div_up(n_groups + g * n_parts, 64), batch), 64, 0, st, (const uint4*)sums, nb, (unsigned)g, col_run, S, P);
  }
  PB_LAUNCH(k_msm_lists, dim3(div_up(plan.nlists, 4), batch, chunks), 128, 0, st, (const uint4*)S, (const uint4*)P, n_groups, n_parts, plan,
            chunks, lists);
  if (chunks > kFinalChunks) {  // S is dead: it takes the folded list sums
    PB_LAUNCH(k_msm_fold, div_up((size_t)batch * plan.nlists, 4), 128, 0, st, (const uint4*)lists, batch * (unsigned)plan.nlists, chunks, S);
    PB_LAUNCH(k_msm_final, batch, 256, 0, st, (const uint4*)S, plan, 1u, result);
  } else {
    PB_LAUNCH(k_msm_final, batch, 256, 0, st, (const uint4*)lists, plan, chunks, result);
  }
  PB_CUDA(cudaGetLastError());
  return 0;
}

// Host tail.  `host` holds n_parts x batch entries of (ndig + 1) XYZZ points (part-major): the digit
// sums of n_parts partial MSMs that share one plan (n_parts = 1 for an ordinary MSM, the rank count for a
// point-sharded one).  R = sum A_G + g * sum_j 2^shift_j D_j is linear in the D_j and in sum A_G, so
// the parts are added digit by digit first and one Horner over the digits follows; then the affine
// normalisation of Commitment::from (commitment.rs:89-93) with one shared inversion per batch
// (Montgomery's trick over the ZZ*ZZZ of the batch's results).
static void msm_finish(const uint32_t* host, const MsmTail& tail, int n_parts, uint64_t* out_affine_host) {
  const DigitPlan& plan = tail.plan;
  const uint32_t batch = tail.batch;
  const size_t wpe = tail.words_per_entry();
  std::vector<pbh::HXyzz> res(batch);
  for (uint32_t b = 0; b < batch; b++) {
    auto digit = [&](int d) {
      pbh::HXyzz s = pbh::HXyzz::identity(), t;
      for (int p = 0; p < n_parts; p++) {
        xyzz_dev_to_host(host + ((size_t)p * batch + b) * wpe + (size_t)d * 48, &t);
        pbh::hxyzz_add(s, t);
      }
      return s;
    };
    pbh::HXyzz h = pbh::HXyzz::identity();
    for (int d = plan.ndig - 1; d >= 0; d--) {
      pbh::HXyzz t = digit(d);
      pbh::hxyzz_add(h, t);
      const int dbl = d > 0 ? plan.bits[d - 1] : tail.log_g;
      for (int k = 0; k < dbl; k++) h = pbh::hxyzz_dbl(h);
    }
    pbh::HXyzz t = digit(plan.ndig);
    pbh::hxyzz_add(h, t);
    res[b] = h;
  }
  std::vector<pbh::HFp> den(batch), pre(batch);
  pbh::HFp acc = pbh::HFp::one();
  for (uint32_t b = 0; b < batch; b++) {
    den[b] = res[b].is_inf() ? pbh::HFp::one() : res[b].zz * res[b].zzz;
    pre[b] = acc;
    acc = acc * den[b];
  }
  pbh::HFp inv = acc.inv();
  for (uint32_t b = batch; b-- > 0;) {
    const pbh::HFp i = inv * pre[b];  // 1 / (zz * zzz)
    inv = inv * den[b];
    pbh::HFp x = pbh::HFp::zero(), y = pbh::HFp::zero();
    if (!res[b].is_inf()) {
      x = res[b].x * (i * res[b].zzz);
      y = res[b].y * (i * res[b].zz);
    }
    memcpy(out_affine_host + (size_t)b * 12, x.v, 48);
    memcpy(out_affine_host + (size_t)b * 12 + 6, y.v, 48);
  }
}

// The host tail on its own (pb200_msm_combine_parts): digit sums of n_parts partial MSMs -> affine results.
int msm_combine_parts(const uint32_t* parts, int n_parts, int window_bits, uint32_t batch, uint64_t* out_affine_host, size_t* words_per_entry) {
  MsmTail tail;
  PB_TRY(msm_plan(window_bits, batch, &tail));
  if (words_per_entry) *words_per_entry = tail.words_per_entry();
  if (parts && out_affine_host) msm_finish(parts, tail, n_parts, out_affine_host);
  return 0;
}

int msm_run(const pb200_srs* srs, size_t first, const uint64_t* d_scalars, size_t n, uint32_t batch, size_t stride,
            MsmShape shape, uint64_t* out_affine_host, cudaStream_t st, Arena* ar) {
  if (first + n > srs->n_points) return fail(PB200_ERR_DEGREE_TOO_LARGE, "more scalars than commit-key points");
  if (batch == 0) return 0;
  if (n == 0) {
    memset(out_affine_host, 0, (size_t)batch * 96);
    return 0;
  }
  const bool prof = g_prof_on.load(std::memory_order_relaxed) != 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  struct EvGuard {
    cudaEvent_t* e;
    ~EvGuard() {
      for (int i = 0; i < 2; i++)
        if (e[i]) cudaEventDestroy(e[i]);
    }
  } ev_guard{ev};
  if (prof) {
    PB_CUDA(cudaEventCreate(&ev[0]));
    PB_CUDA(cudaEventCreate(&ev[1]));
  }
  ScratchScope scope(ar, st);
  uint4* result = nullptr;
  MsmTail tail;
  const unsigned* d_totals = nullptr;
  PB_TRY(msm_enqueue(srs, first, d_scalars, n, batch, stride, shape, st, scope, &result, &tail, prof ? ev : nullptr, &d_totals));
  std::vector<unsigned> h_tot(batch, 0);
  if (prof) {
    const unsigned nb = 1u << (srs->c - 1);
    PB_CUDA(cudaMemcpy2DAsync(h_tot.data(), 4, d_totals, (size_t)(nb + 1) * 4, 4, batch, cudaMemcpyDeviceToHost, st));
  }
  const size_t host_words = (size_t)batch * tail.words_per_entry();
  uint32_t* host = (uint32_t*)pinned_scratch(host_words * 4);
  if (!host) return fail(PB200_ERR_CUDA, "pinned staging buffer");
  PB_CUDA(cudaMemcpyAsync(host, result, host_words * 4, cudaMemcpyDeviceToHost, st));
  PB_CUDA(stream_wait(st));
  if (prof) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) {
      uint64_t adds = 0;
      for (unsigned t : h_tot) adds += t;
      const bool sparse = adds * 4 < (uint64_t)n * batch * srs->W;
      (sparse ? g_prof_sp_ns : g_prof_acc_ns).fetch_add((uint64_t)(ms * 1e6));
      (sparse ? g_prof_sp_adds : g_prof_acc_adds).fetch_add(adds);
      (sparse ? g_prof_sp_points : g_prof_acc_points).fetch_add((uint64_t)n * batch);
      (sparse ? g_prof_sp_launches : g_prof_acc_launches).fetch_add(1);
    }
  }
  scope.release();  // the stream was synchronised above: the scratch is dead
  msm_finish(host, tail, 1, out_affine_host);
  return 0;
}

// ---- point-sharded MSM: slice MSM -> ONE ncclAllGather of the digit sums -> local sum (SURVEY.md
// section 8e-ii, BASELINE configs[3]).  The gather runs on device buffers on the MSM's own stream,
// straight behind the reduction kernels: there is one host synchronisation per call.  Every rank's
// record starts with a 16-byte header {status, c, ndig, batch}; a rank whose local part failed still
// joins the collective with status != 0, so its peers return an error instead of hanging.
int msm_allgather(const pb200_srs* srs, const uint64_t* scalars, bool scalars_on_device, size_t n, uint32_t batch, size_t stride,
                  nccl_all_gather_fn all_gather, void* comm, int n_ranks, int* nccl_rc, uint64_t* out_affine_host, cudaStream_t st) {
  MsmTail tail;
  PB_TRY(msm_plan(srs->c, batch, &tail));
  const size_t payload = (size_t)batch * tail.words_per_entry() * 4, rec = 16 + payload;
  ScratchScope scope(nullptr, st);
  uint8_t *d_send = nullptr, *d_recv = nullptr;
  PB_ALLOC(scope, d_send, rec);
  PB_ALLOC(scope, d_recv, rec * (size_t)n_ranks);
  uint8_t* host = (uint8_t*)pinned_scratch(rec * (size_t)n_ranks + 16);
  if (!host) return fail(PB200_ERR_CUDA, "pinned staging buffer");
  uint32_t* hdr = (uint32_t*)(host + rec * (size_t)n_ranks);  // staging for this rank's header
  // local part; from here on every path reaches the collective
  int local_rc = 0;
  {
    uint4* result = nullptr;
    MsmTail t2;
    const uint64_t* d_scalars = scalars;
    if (!scalars_on_device && n) {
      uint64_t* d = (uint64_t*)scope.take((size_t)batch * n * 32);
      cudaError_t e = d ? cudaMemcpy2DAsync(d, n * 32, scalars, stride * 32, n * 32, batch, cudaMemcpyHostToDevice, st) : cudaErrorMemoryAllocation;
      if (e != cudaSuccess) local_rc = fail(PB200_ERR_CUDA, "scalar upload", cudaGetErrorString(e));
      d_scalars = d;
      stride = n;
    }
    if (local_rc == 0) local_rc = msm_enqueue(srs, 0, d_scalars, n, batch, stride, kMsmLatency, st, scope, &result, &t2, nullptr, nullptr);
    cudaError_t e = cudaSuccess;
    if (local_rc == 0) e = cudaMemcpyAsync(d_send + 16, result, payload, cudaMemcpyDeviceToDevice, st);
    if (local_rc != 0 || e != cudaSuccess) {
      if (local_rc == 0) local_rc = fail(PB200_ERR_CUDA, "partial result copy", cudaGetErrorString(e));
      cudaMemsetAsync(d_send + 16, 0, payload, st);
    }
  }
  const std::string local_msg = g_last_error;
  hdr[0] = local_rc ? 1u : 0u;
  hdr[1] = (uint32_t)tail.c;
  hdr[2] = (uint32_t)tail.plan.ndig;
  hdr[3] = batch;
  cudaError_t e = cudaMemcpyAsync(d_send, hdr, 16, cudaMemcpyHostToDevice, st);
  *nccl_rc = 0;
  if (e == cudaSuccess) *nccl_rc = all_gather(d_send, d_recv, rec, /*ncclUint8*/ 1, comm, st);
  if (e == cudaSuccess && *nccl_rc == 0) e = cudaMemcpyAsync(host, d_recv, rec * (size_t)n_ranks, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && *nccl_rc == 0) e = stream_wait(st);
  if (*nccl_rc != 0) return fail(PB200_ERR_CUDA, "ncclAllGather");
  PB_CUDA(e);
  scope.release();
  if (local_rc != 0) {
    g_last_error = local_msg;
    return local_rc;
  }
  std::vector<uint32_t> parts((size_t)n_ranks * payload / 4);
  for (int r = 0; r < n_ranks; r++) {
    const uint32_t* h = (const uint32_t*)(host + rec * (size_t)r);
    if (h[0] != 0) {
      char msg[48];
      snprintf(msg, sizeof msg, "rank %d", r);
      return fail(PB200_ERR_CUDA, "the partial MSM of another rank failed", msg);
    }
    if (h[1] != (uint32_t)tail.c || h[2] != (uint32_t)tail.plan.ndig || h[3] != batch)
      return fail(PB200_ERR_INVALID_ARG, "ranks disagree on the MSM window or batch (key slices must use one window width)");
    memcpy(parts.data() + (size_t)r * payload / 4, h + 4, payload);
  }
  msm_finish(parts.data(), tail, n_ranks, out_affine_host);
  return 0;
}

// The arena bytes one msm_run(n, batch) call carves, in either shape.
size_t msm_workspace_bytes(const pb200_srs* srs, size_t n, uint32_t batch) {
  MsmScratch s;
  if (msm_scratch(srs->c, srs->W, n, batch, msm_affine_enabled(), &s) != 0) return 0;
  size_t total = 0;
  for (size_t b : s.bytes) total += Arena::round_up(b);
  return total;
}

// The windows w >= 1 of a table whose window 0 is on the device, and whether any entry is the identity.
static cudaError_t srs_fill_windows(pb200_srs* s, cudaStream_t st) {
  unsigned* d_inf = nullptr;
  unsigned n_inf = 0;
  cudaError_t e = cudaMalloc((void**)&d_inf, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemsetAsync(d_inf, 0, sizeof(unsigned), st);
  if (e == cudaSuccess) {
    PB_LAUNCH(k_msm_precompute, div_up(s->n_points, 64), 64, 0, st, s->table, s->n_points, s->c, s->W, d_inf);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&n_inf, d_inf, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(d_inf);
  s->has_inf = n_inf != 0;
  return e;
}

int srs_upload(const uint8_t* raw, size_t n_points, pb200_srs** out, int window_bits) {
  if (n_points == 0) return fail(PB200_ERR_INVALID_ARG, "empty commit key");
  cudaStream_t st = thread_stream();
  pb200_srs* s = new pb200_srs();
  s->n_points = n_points;
  s->c = window_bits ? window_bits : pick_window(n_points);
  s->W = (256 + s->c - 1) / s->c;
  s->table = nullptr;
  cudaError_t e = cudaMalloc((void**)&s->table, (size_t)s->W * n_points * 96);
  if (e != cudaSuccess) {
    delete s;
    return fail(PB200_ERR_CUDA, "cudaMalloc(commit key table)", cudaGetErrorString(e));
  }
  e = cudaMemcpyAsync(s->table, raw, n_points * 96, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = srs_fill_windows(s, st);
  if (e != cudaSuccess) {
    cudaFree(s->table);
    delete s;
    return fail(PB200_ERR_CUDA, "commit key upload", cudaGetErrorString(e));
  }
  *out = s;
  return 0;
}

// The key's points as uploaded (window 0 of the table), n_points affine points on the device.
const uint4* srs_points(const pb200_srs* s) { return s->table; }

// srs_upload for points that are already on the device (e.g. the Lagrange form made by csrc/ecntt.cu).
int srs_from_device(const uint4* d_points, size_t n_points, pb200_srs** out, int window_bits) {
  if (n_points == 0) return fail(PB200_ERR_INVALID_ARG, "empty commit key");
  cudaStream_t st = thread_stream();
  pb200_srs* s = new pb200_srs();
  s->n_points = n_points;
  s->c = window_bits ? window_bits : pick_window(n_points);
  s->W = (256 + s->c - 1) / s->c;
  s->table = nullptr;
  cudaError_t e = cudaMalloc((void**)&s->table, (size_t)s->W * n_points * 96);
  if (e != cudaSuccess) {
    delete s;
    return fail(PB200_ERR_CUDA, "cudaMalloc(commit key table)", cudaGetErrorString(e));
  }
  e = cudaMemcpyAsync(s->table, d_points, n_points * 96, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = srs_fill_windows(s, st);
  if (e != cudaSuccess) {
    cudaFree(s->table);
    delete s;
    return fail(PB200_ERR_CUDA, "commit key table", cudaGetErrorString(e));
  }
  *out = s;
  return 0;
}

// The generator's window table of k_srs_setup, built on first use and kept for the life of the process.
static int srs_gen_table(const uint4** out) {
  static std::once_flag once;
  static uint4* table = nullptr;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [] {
    cudaStream_t st = thread_stream();
    err = cudaMalloc((void**)&table, (size_t)kSetupW * kSetupHalf * 96);
    if (err == cudaSuccess) {
      PB_LAUNCH(k_srs_gen_table, div_up(kSetupW * kSetupHalf, 128), 128, 0, st, table);
      err = cudaGetLastError();
    }
    if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  });
  if (err != cudaSuccess) return fail(PB200_ERR_CUDA, "generator table for the commit-key setup", cudaGetErrorString(err));
  *out = table;
  return 0;
}

int srs_setup_dev(const uint64_t* x_mont, const uint64_t* g_scalar_mont, size_t n, uint4* d_out) {
  const uint4* table = nullptr;
  PB_TRY(srs_gen_table(&table));
  cudaStream_t st = thread_stream();
  // Runs of up to 32 points share an inversion; shorter runs keep about 1024 threads per SM busy on small keys.
  const size_t want_threads = (size_t)std::max(1u, num_sms()) * 1024;
  const unsigned run = (unsigned)std::min<size_t>(32, std::max<size_t>(1, div_up(n, want_threads)));
  const size_t threads = div_up(div_up(n, run), 128) * 128;
  uint4* scratch = nullptr;  // a plain allocation: a large key's scratch does not stay in the stream pool
  cudaError_t e = cudaMalloc((void**)&scratch, (size_t)run * threads * 96);
  Fr x, gs;
  memcpy(x.v, x_mont, 32);
  memcpy(gs.v, g_scalar_mont, 32);
  if (e == cudaSuccess) {
    PB_LAUNCH(k_srs_setup, threads / 128, 128, 0, st, d_out, n, x, gs, table, scratch, run);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(scratch);
  PB_CUDA(e);
  return 0;
}

int srs_setup(const uint64_t* x_mont, const uint64_t* g_scalar_mont, size_t n, uint8_t* out_raw) {
  uint4* d = nullptr;
  PB_CUDA(cudaMalloc((void**)&d, n * 96));
  int rc = srs_setup_dev(x_mont, g_scalar_mont, n, d);
  if (rc == 0) {
    const cudaError_t e = cudaMemcpy(out_raw, d, n * 96, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) rc = fail(PB200_ERR_CUDA, "commit-key setup copy", cudaGetErrorString(e));
  }
  cudaFree(d);
  return rc;
}

int g1_decompress(const uint8_t* in, size_t n, int check_subgroup, uint8_t* out_raw) {
  cudaStream_t st = thread_stream();
  uint8_t* d_in = nullptr;
  uint4* d_out = nullptr;
  unsigned* d_bad = nullptr;
  PB_CUDA(cudaMalloc((void**)&d_in, n * 48));
  PB_CUDA(cudaMalloc((void**)&d_out, n * 96));
  PB_CUDA(cudaMalloc((void**)&d_bad, 4));
  unsigned bad = 0xffffffffu;
  cudaError_t e = cudaMemcpyAsync(d_in, in, n * 48, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0xff, 4, st);
  if (e == cudaSuccess) {
    PB_LAUNCH(k_g1_decompress, div_up(n, 64), 64, 0, st, d_in, n, check_subgroup, d_out, d_bad);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_raw, d_out, n * 96, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(d_in);
  cudaFree(d_out);
  cudaFree(d_bad);
  PB_CUDA(e);
  if (bad != 0xffffffffu) {
    char msg[64];
    snprintf(msg, sizeof msg, "point %u", bad);
    return fail(PB200_ERR_POINT_MALFORMED, "malformed G1 encoding (not canonical, not on the curve or not in the subgroup)", msg);
  }
  return 0;
}

// The same decoding on device buffers, enqueued on `st`: the verifier decodes the commitments of a batch of
// proofs and tells malformed points from the identity by their encodings.
void g1_decompress_dev(const uint8_t* d_in, size_t n, uint4* d_out, unsigned* d_bad, cudaStream_t st) {
  PB_LAUNCH(k_g1_decompress, div_up(n, 64), 64, 0, st, d_in, n, 1, d_out, d_bad);
}

int g1_check_raw(const uint8_t* raw, size_t n) {
  if (!n) return 0;
  cudaStream_t st = thread_stream();
  uint4* d = nullptr;
  unsigned* d_bad = nullptr;
  PB_CUDA(cudaMalloc((void**)&d, n * 96));
  cudaError_t e = cudaMalloc((void**)&d_bad, 4);
  unsigned bad = 0xffffffffu;
  if (e == cudaSuccess) e = cudaMemcpyAsync(d, raw, n * 96, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0xff, 4, st);
  if (e == cudaSuccess) {
    PB_LAUNCH(k_g1_check_raw, div_up(n, 64), 64, 0, st, (const uint4*)d, n, d_bad);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(d);
  cudaFree(d_bad);
  PB_CUDA(e);
  if (bad != 0xffffffffu) {
    char msg[64];
    snprintf(msg, sizeof msg, "point %u", bad);
    return fail(PB200_ERR_POINT_MALFORMED, "commit-key point not on the curve or not in the prime-order subgroup (PointMalformed)", msg);
  }
  return 0;
}

// n raw points (host) -> n x 48 compressed bytes (host): CommitKey::to_var_bytes
int g1_compress_batch(const uint8_t* raw, size_t n, uint8_t* out_48) {
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint4 *d_in = nullptr, *d_out = nullptr;
  PB_ALLOC(scope, d_in, n * 96);
  PB_ALLOC(scope, d_out, n * 48);
  PB_CUDA(cudaMemcpyAsync(d_in, raw, n * 96, cudaMemcpyHostToDevice, st));
  PB_LAUNCH(k_g1_compress, div_up(n, 128), 128, 0, st, (const uint4*)d_in, n, d_out);
  PB_CUDA(cudaGetLastError());
  PB_CUDA(cudaMemcpyAsync(out_48, d_out, n * 48, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int selftest_mul(int which, const uint64_t* a, const uint64_t* b, uint64_t* o, size_t n) {
  cudaStream_t st = thread_stream();
  const size_t bytes = n * (which ? 48 : 32);
  uint4 *da, *db, *dout;
  PB_CUDA(cudaMalloc((void**)&da, bytes));
  PB_CUDA(cudaMalloc((void**)&db, bytes));
  PB_CUDA(cudaMalloc((void**)&dout, bytes));
  PB_CUDA(cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, st));
  if (which)
    PB_LAUNCH(k_selftest_fp_mul, div_up(n, 128), 128, 0, st, da, db, dout, n);
  else
    PB_LAUNCH(k_selftest_fr_mul, div_up(n, 128), 128, 0, st, da, db, dout, n);
  PB_CUDA(cudaMemcpyAsync(o, dout, bytes, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  cudaFree(da); cudaFree(db); cudaFree(dout);
  return 0;
}

int selftest_fp_ops(const uint64_t* a, const uint64_t* b, const uint64_t* c, const uint64_t* d, uint64_t* o, size_t n) {
  cudaStream_t st = thread_stream();
  const size_t bytes = n * 48;
  uint4* buf;  // a | b | c | d | three outputs
  PB_CUDA(cudaMalloc((void**)&buf, 7 * bytes));
  const uint64_t* in[4] = {a, b, c, d};
  for (int k = 0; k < 4; k++) {
    cudaError_t e = cudaMemcpyAsync((char*)buf + k * bytes, in[k], bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(buf); PB_CUDA(e); }
  }
  uint4* p = buf;
  const size_t q = bytes / 16;
  if (n) PB_LAUNCH(k_selftest_fp_ops, div_up(n, 128), 128, 0, st, p, p + q, p + 2 * q, p + 3 * q, p + 4 * q, n);
  cudaError_t e = cudaMemcpyAsync(o, (char*)buf + 4 * bytes, 3 * bytes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(buf);
  PB_CUDA(e);
  return 0;
}

int imad_peak(double* out) {
  cudaStream_t st = thread_stream();
  unsigned* d;
  PB_CUDA(cudaMalloc((void**)&d, 4));
  cudaDeviceProp prop;
  int dev;
  PB_CUDA(cudaGetDevice(&dev));
  PB_CUDA(cudaGetDeviceProperties(&prop, dev));
  const int blocks = prop.multiProcessorCount * 8, threads = 256, iters = 2000;
  PB_LAUNCH(k_imad_peak, blocks, threads, 0, st, d, 50, 1u);
  cudaEvent_t e0, e1;
  PB_CUDA(cudaEventCreate(&e0));
  PB_CUDA(cudaEventCreate(&e1));
  PB_CUDA(cudaEventRecord(e0, st));
  PB_LAUNCH(k_imad_peak, blocks, threads, 0, st, d, iters, 2u);
  PB_CUDA(cudaEventRecord(e1, st));
  PB_CUDA(cudaStreamSynchronize(st));
  float ms = 0;
  PB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *out = (double)blocks * threads * iters * 64.0 / (ms * 1e-3);
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
  return 0;
}

int fp_product_peak(double* out) {
  cudaStream_t st = thread_stream();
  uint4* d;
  PB_CUDA(cudaMalloc((void**)&d, 48));
  cudaDeviceProp prop;
  int dev;
  PB_CUDA(cudaGetDevice(&dev));
  PB_CUDA(cudaGetDeviceProperties(&prop, dev));
  const int blocks = prop.multiProcessorCount * 4, threads = 256, iters = 400;
  PB_LAUNCH(k_fp_product_peak, blocks, threads, 0, st, d, 20, 1u);
  cudaEvent_t e0, e1;
  PB_CUDA(cudaEventCreate(&e0));
  PB_CUDA(cudaEventCreate(&e1));
  PB_CUDA(cudaEventRecord(e0, st));
  PB_LAUNCH(k_fp_product_peak, blocks, threads, 0, st, d, iters, 2u);
  PB_CUDA(cudaEventRecord(e1, st));
  PB_CUDA(cudaStreamSynchronize(st));
  float ms = 0;
  PB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *out = (double)blocks * threads * iters * 2.0 / (ms * 1e-3);
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
  return 0;
}

}  // namespace pb

namespace pb {
size_t srs_len(const pb200_srs* s) { return s->n_points; }
int srs_window(const pb200_srs* s) { return s->c; }
int msm_window_for(size_t n_points) { return pick_window(n_points ? n_points : 1); }
void srs_free(pb200_srs* s) {
  cudaFree(s->table);
  delete s;
}
}  // namespace pb
