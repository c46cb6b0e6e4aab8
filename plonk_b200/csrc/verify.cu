// Verifier (reference src/compiler/verifier.rs): Verifier::verify_with_version for a batch of proofs per call, one
// verdict per proof, for PlonkVersion V1, V2 and V3.
//
// The host parses, replays the transcript and computes the O(#public inputs) scalars of Proof::verify
// (src/proof_system/proof.rs:218-516) or, for V1, Proof::verify_legacy (proof.rs:518-790); see verify_scalars.h.
// The device decodes the commitments (k_g1_decompress), forms the two G1 points of the final pairing check with one
// warp per proof (k_verify_msm), and runs the multi-Miller loop, the final exponentiation and the comparison with 1
// with one thread per proof (k_verify_pairing).  The device work is the same for every version: V1 only gives the
// four selector-opening terms zero scalars.
//
// Batch verification (pb200_batch_verify_groups, and pb200_batch_verify as its one-group case) gives one verdict for
// groups of proofs under verifiers that share one opening key, with one pairing: the host draws rho from the groups'
// versions, lengths and u challenges (verify_scalars.h), k_batch_fold weighs each proof's terms by w_i = rho^i and sums
// the verifier-key terms per key slot (one slot per distinct verifier), k_batch_msm / k_batch_reduce form
// sum w_i L_i and sum w_i R_i, and k_verify_pairing checks the pair.
#include <algorithm>
#include <mutex>
#include <numeric>
#include <thread>
#include <unordered_map>
#include <vector>

#include "internal.cuh"
#include "g1.cuh"
#include "host_field.h"
#include "pairing.cuh"
#include "plonk_algebra.cuh"
#include "transcript.h"
#include "verify_scalars.h"

struct pb200_verifier {
  std::vector<uint8_t> label;
  uint64_t vk_n = 0;                          // VerifierKey::n: the constraint count for a compiled circuit
  uint64_t size = 0, constraints = 0;         // Verifier::size, Verifier::constraints
  uint8_t vk_comm[pb::N_POLY][48];             // pb::Poly order
  uint8_t opening_key[PB200_OPENING_KEY_BYTES];
  std::vector<uint64_t> pi_idx;
  pb::VerifyKeyHost key;            // both base transcripts, the domain (EvaluationDomain::new(vk_n)) and the pi roots
  uint4* d_points = nullptr;        // the 15 key commitments then opening_key.g, 96-byte raw affine
  pb::LineCoeffs* d_lines = nullptr;  // prepared [x]H then H, PB_G2_LINES each
};

namespace pb {
namespace {
using pbh::HFr;

PB_D G1Affine ld_aff(const uint4* q) {
  G1Affine p;
  const uint32_t* w = (const uint32_t*)q;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    p.x.v[k] = w[k];
    p.y.v[k] = w[12 + k];
  }
  return p;
}
PB_D void st_aff(uint4* q, const G1Affine& p) {
  uint32_t* w = (uint32_t*)q;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    w[k] = p.x.v[k];
    w[12 + k] = p.y.v[k];
  }
}
PB_D G1Xyzz shfl_down_xyzz(const G1Xyzz& a, int d) {
  G1Xyzz r;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    r.x.v[k] = __shfl_down_sync(0xffffffffu, a.x.v[k], d);
    r.y.v[k] = __shfl_down_sync(0xffffffffu, a.y.v[k], d);
    r.zz.v[k] = __shfl_down_sync(0xffffffffu, a.zz.v[k], d);
    r.zzz.v[k] = __shfl_down_sync(0xffffffffu, a.zzz.v[k], d);
  }
  return r;
}
PB_D G1Affine to_affine(const G1Xyzz& p) {
  if (p.is_inf()) return {Fp::zero(), Fp::zero()};
  const Fp zz = p.zz.canonical(), zzz = p.zzz.canonical();
  const Fp i = fp_inv_bingcd(zz * zzz);
  return {p.x.canonical() * (i * zzz), p.y.canonical() * (i * zz)};
}

// Lane k of a warp multiplies term k of right_projective (proof.rs:300-455): the source of its point is a key
// point (0..15: the 15 commitments in pb200_prover_commitments order, then opening_key.g) or a proof commitment
// (16 + its index in Proof::to_bytes order); -1 = no term.  Lane 31 computes u [W_zw] + [W_z] for left_projective.
enum { P_A = 16, P_B, P_C, P_D, P_Z, P_TLOW, P_TMID, P_THIGH, P_TFOURTH, P_WZ, P_WZW };
__constant__ int c_term_point[32] = {0,  1,  2,  3,       4,      5,      7,       8,         9,    10, P_Z,   14, P_TLOW, P_TMID, P_THIGH, P_TFOURTH,
                                     P_A, P_B, P_C, P_D, 11, 12, 13, 6, 5, 1, 2, 15, P_WZ, P_WZW, -1, P_WZW};

// Whether proof i has a malformed commitment, evaluated by a whole warp (lane k tests commitment k).  k_g1_decompress
// leaves zeros for an encoding it rejects (not canonical, not on the curve or not torsion-free), so a commitment
// that decoded to zeros without being the identity's encoding is malformed.  proof_comm: [proof][11] compressed
// commitments; pts: their decoded points.
PB_D bool warp_proof_malformed(const uint4* pts, const uint8_t* proof_comm, size_t i, int lane) {
  bool bad = false;
  if (lane < 11) {
    const uint4* q = pts + 6 * (i * 11 + lane);
    const G1Affine p = ld_aff(q);
    if (p.is_inf()) {
      const uint8_t* e = proof_comm + 48 * (i * 11 + lane);
      uint32_t acc = e[0] ^ 0xc0u;
      for (int k = 1; k < 48; k++) acc |= e[k];
      bad = acc != 0;
    }
  }
  return __any_sync(0xffffffffu, bad);
}

// One warp per proof.  scalars: [proof][32] canonical little-endian Fr; proof_comm, pts: as warp_proof_malformed.
// status: PB200_OK on entry or the host's verdict.  out: [proof] -(W_z + u W_zw), right.
__global__ void __launch_bounds__(128) k_verify_msm(const uint4* key_pts, const uint4* pts, const uint8_t* proof_comm,
                                                    const uint4* scalars, size_t n, int* status, uint4* out) {
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;  // whole warps
  if (warp_proof_malformed(pts, proof_comm, i, lane)) {
    if (lane == 0) status[i] = PB200_ERR_POINT_MALFORMED;
    return;
  }
  if (status[i] != PB200_OK) return;
  G1Xyzz acc = G1Xyzz::identity();
  const int src = c_term_point[lane];
  if (src >= 0) {
    const G1Affine p = src < 16 ? ld_aff(key_pts + 6 * src) : ld_aff(pts + 6 * (i * 11 + (src - 16)));
    if (!p.is_inf()) {
      const uint4* sp = scalars + 2 * (i * PB_VERIFY_TERMS + lane);
      const uint4 lo = sp[0], hi = sp[1];
      const uint32_t s[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll 1
      for (int w = 7; w >= 0; w--) {
#pragma unroll 1
        for (int b = 31; b >= 0; b--) {
          acc = xyzz_dbl(acc);
          if ((s[w] >> b) & 1u) xyzz_madd(acc, p.x, p.y);
        }
      }
    }
  }
  G1Xyzz left = G1Xyzz::identity();
  if (lane == 31) {
    const G1Affine wz = ld_aff(pts + 6 * (i * 11 + (P_WZ - 16)));
    left = acc;
    if (!wz.is_inf()) xyzz_madd(left, wz.x, wz.y);
    left = left.neg();
    acc = G1Xyzz::identity();
  }
#pragma unroll 1
  for (int d = 16; d >= 1; d >>= 1) {
    const G1Xyzz o = shfl_down_xyzz(acc, d);
    xyzz_add(acc, o);
  }
  if (lane == 0) st_aff(out + 12 * i + 6, to_affine(acc));
  if (lane == 31) st_aff(out + 12 * i, to_affine(left));
}

// One thread per proof: e(-(W_z + u W_zw), [x]H) e(right, H) == 1 (proof.rs:498-513).
__global__ void __launch_bounds__(64) k_verify_pairing(const uint4* g1, const LineCoeffs* lines, size_t n, int* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || status[i] != PB200_OK) return;
  G1Affine p[2] = {ld_aff(g1 + 12 * i), ld_aff(g1 + 12 * i + 6)};
  const LineCoeffs* l[2] = {lines, lines + PB_G2_LINES};
  const Fp12 f = final_exponentiation(miller_loop2(p, l));
  status[i] = f.is_one() ? PB200_OK : PB200_ERR_VERIFY;
}

// ---- batch verification -----------------------------------------------------------------------------------------
// Proof i's check is e(L_i, [x]H) e(R_i, H) = 1 with L_i = -(W_z + u_i W_zw) and R_i = sum_k s_ik P_ik, the 31 terms
// of k_verify_msm's lanes 0..30.  The batch's check is the same with L = sum w_i L_i and R = sum w_i R_i, formed as
// two dense term lists: R has the 11 proof commitments of every proof (term 11 i + j is commitment j of proof i, so
// its point is pts[11 i + j]) followed by 16 key points per key slot (term 11 n + 16 s + k is key point k of slot s,
// read from the gathered table key_pts[16 s + k]), whose scalars are summed over the slot's proofs; L has W_z and
// W_zw of every proof (terms 2 i and 2 i + 1) and is negated once at the end.
constexpr int kBatchFoldWarps = 8;  // proofs per block of k_batch_fold

// A block of k_batch_fold: proofs [first, first + count), count <= kBatchFoldWarps, all under one key slot.
struct FoldBlock {
  uint32_t first, count;
};

PB_D Fr ld_fr(const uint4* q) {
  Fr x;
  const uint4 lo = q[0], hi = q[1];
  x.v[0] = lo.x, x.v[1] = lo.y, x.v[2] = lo.z, x.v[3] = lo.w;
  x.v[4] = hi.x, x.v[5] = hi.y, x.v[6] = hi.z, x.v[7] = hi.w;
  return x;
}
PB_D void st_fr(uint4* q, const Fr& x) {
  q[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
  q[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}

// One warp per proof, lane k on term k of k_verify_msm.  weights: [proof] w_i (Montgomery form, so that w_i times a
// canonical scalar is canonical); status: the host's verdicts.  A proof that the host or the decoder rejected gets
// weight 0 and sets flags (bit 0: malformed, bit 1: fails the check).  Writes the 11 n proof-term scalars of R
// (r_scal) and the 2 n scalars of L (l_scal: w_i, w_i u_i), and per block the sums over its proofs of the 19
// key-point lanes, merged into the 16 key points (key_part: [block][16]).  blocks: which proofs each block takes;
// the host lists the blocks slot by slot, so that a slot's partial sums are one contiguous range.
__global__ void __launch_bounds__(32 * kBatchFoldWarps) k_batch_fold(const uint4* pts, const uint8_t* proof_comm, const uint4* scalars,
                                                                    const uint4* weights, const int* status, const FoldBlock* blocks,
                                                                    unsigned* flags, uint4* r_scal, uint4* l_scal, uint4* key_part) {
  __shared__ uint4 part[kBatchFoldWarps][32][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const FoldBlock blk = blocks[blockIdx.x];
  const size_t i = (size_t)blk.first + warp;
  const int src = c_term_point[lane];
  Fr prod = Fr::zero();
  if (warp < (int)blk.count) {  // whole warps
    const bool bad = warp_proof_malformed(pts, proof_comm, i, lane);
    const int st = bad ? PB200_ERR_POINT_MALFORMED : status[i];
    if (lane == 0 && st != PB200_OK) atomicOr(flags, st == PB200_ERR_POINT_MALFORMED ? 1u : 2u);
    const Fr w = st == PB200_OK ? ld_fr(weights + 2 * i) : Fr::zero();
    prod = w * ld_fr(scalars + 2 * (i * PB_VERIFY_TERMS + lane));
    if (lane == 31) {  // u: left's W_zw term
      st_fr(l_scal + 2 * (2 * i), w.from_mont());
      st_fr(l_scal + 2 * (2 * i + 1), prod);
    } else if (src >= 16) {
      st_fr(r_scal + 2 * (i * 11 + (src - 16)), prod);
    }
  }
  st_fr(part[warp][lane], prod);
  __syncthreads();
  if (threadIdx.x < 16) {
    Fr acc = Fr::zero();
    for (int l = 0; l < 31; l++)
      if (c_term_point[l] == (int)threadIdx.x)
        for (int w = 0; w < kBatchFoldWarps; w++) acc = acc + ld_fr(part[w][l]);
    st_fr(key_part + 2 * ((size_t)blockIdx.x * 16 + threadIdx.x), acc);
  }
}

// Block 16 s + k sums key point k's partial scalars over slot s's blocks of k_batch_fold, [slot_blocks[s],
// slot_blocks[s + 1]), into r_keys[16 s + k]; block 0 turns the flags into the verdict (malformed before a failed
// check).
__global__ void __launch_bounds__(256) k_batch_key_sums(const uint4* key_part, const uint32_t* slot_blocks, const unsigned* flags,
                                                        int* verdict, uint4* r_keys) {
  __shared__ uint4 s[256][2];
  const uint32_t slot = blockIdx.x >> 4, k = blockIdx.x & 15;
  Fr acc = Fr::zero();
  for (size_t b = slot_blocks[slot] + threadIdx.x; b < slot_blocks[slot + 1]; b += 256) acc = acc + ld_fr(key_part + 2 * (b * 16 + k));
  st_fr(s[threadIdx.x], acc);
  __syncthreads();
  for (int d = 128; d >= 1; d >>= 1) {
    if ((int)threadIdx.x < d) st_fr(s[threadIdx.x], ld_fr(s[threadIdx.x]) + ld_fr(s[threadIdx.x + d]));
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    st_fr(r_keys + 2 * blockIdx.x, ld_fr(s[0]));
    if (blockIdx.x == 0) *verdict = (*flags & 1u) ? PB200_ERR_POINT_MALFORMED : (*flags & 2u) ? PB200_ERR_VERIFY : PB200_OK;
  }
}

// One lane per term, 32 terms per warp: threads [0, r_pad) take R's n_r terms (the first n_proof_terms of them proof
// commitments, the rest key points), threads [r_pad, r_pad + l_pad) take L's n_l terms (both lists padded to whole
// warps with empty terms).  Per-lane double-and-add in XYZZ as in k_verify_msm, then a warp sum; partial[warp]
// receives it.  Nothing runs once the verdict is a failure.
__global__ void __launch_bounds__(128) k_batch_msm(const uint4* key_pts, const uint4* pts, const uint4* r_scal, size_t n_proof_terms,
                                                   size_t n_r, size_t r_pad, const uint4* l_scal, size_t n_l, size_t l_pad,
                                                   const int* verdict, G1Xyzz* partial) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= r_pad + l_pad || *verdict != PB200_OK) return;  // whole warps
  const bool is_r = t < r_pad;
  const size_t k = is_r ? t : t - r_pad;
  G1Xyzz acc = G1Xyzz::identity();
  if (k < (is_r ? n_r : n_l)) {
    const G1Affine p = !is_r ? ld_aff(pts + 6 * ((k >> 1) * 11 + (P_WZ - 16) + (k & 1)))
                       : k < n_proof_terms ? ld_aff(pts + 6 * k)
                                           : ld_aff(key_pts + 6 * (k - n_proof_terms));
    if (!p.is_inf()) {
      const uint4* sp = (is_r ? r_scal : l_scal) + 2 * k;
      const uint4 lo = sp[0], hi = sp[1];
      const uint32_t s[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll 1
      for (int w = 7; w >= 0; w--) {
#pragma unroll 1
        for (int b = 31; b >= 0; b--) {
          acc = xyzz_dbl(acc);
          if ((s[w] >> b) & 1u) xyzz_madd(acc, p.x, p.y);
        }
      }
    }
  }
#pragma unroll 1
  for (int d = 16; d >= 1; d >>= 1) {
    const G1Xyzz o = shfl_down_xyzz(acc, d);
    xyzz_add(acc, o);
  }
  if ((threadIdx.x & 31) == 0) partial[t >> 5] = acc;
}

// Block 0 sums R's r_warps warp partials, block 1 the l_warps after them and negates; out: L then R, 96-byte raw
// affine each, the layout k_verify_pairing reads.
__global__ void __launch_bounds__(256) k_batch_reduce(const G1Xyzz* partial, size_t r_warps, size_t l_warps, const int* verdict,
                                                      uint4* out) {
  __shared__ G1Xyzz s[8];
  if (*verdict != PB200_OK) return;
  const bool is_r = blockIdx.x == 0;
  const G1Xyzz* p = is_r ? partial : partial + r_warps;
  const size_t m = is_r ? r_warps : l_warps;
  G1Xyzz acc = G1Xyzz::identity();
#pragma unroll 1
  for (size_t k = threadIdx.x; k < m; k += 256) xyzz_add(acc, p[k]);
#pragma unroll 1
  for (int d = 16; d >= 1; d >>= 1) {
    const G1Xyzz o = shfl_down_xyzz(acc, d);
    xyzz_add(acc, o);
  }
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll 1
    for (int w = 1; w < 8; w++) xyzz_add(acc, s[w]);
    st_aff(out + (is_r ? 6 : 0), to_affine(is_r ? acc : acc.neg()));
  }
}

// Decodes `count` G2 points (96-byte encodings) and prepares the lines of each non-identity one.  ok[k]: 1 for a
// valid encoding of a non-identity point, 2 for the identity, 0 for a rejected encoding.
__global__ void k_g2_prepare(const uint8_t* enc, int count, LineCoeffs* lines, int* ok) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  G2Affine q;
  const bool valid = g2_decode(enc + 96 * k, &q);
  ok[k] = !valid ? 0 : (q.inf ? 2 : 1);
  if (valid && !q.inf && lines) g2_prepare(q, lines + (size_t)PB_G2_LINES * k);
}

// The G2 half of PublicParameters::setup (srs.rs:91-93): h = [h_scalar] G2Affine::generator() and x_h = [x] h, written
// as two 96-byte compressed points (h, then x_h).  Scalars in Montgomery form.  One thread: two scalar multiplications.
__global__ void k_opening_key_g2(Fr x, Fr h_scalar, uint8_t* out) {
  if (blockIdx.x || threadIdx.x) return;
  const uint8_t gen[96] = {  // G2Affine::generator().to_compressed()
      0x93, 0xe0, 0x2b, 0x60, 0x52, 0x71, 0x9f, 0x60, 0x7d, 0xac, 0xd3, 0xa0, 0x88, 0x27, 0x4f, 0x65, 0x59, 0x6b, 0xd0, 0xd0,
      0x99, 0x20, 0xb6, 0x1a, 0xb5, 0xda, 0x61, 0xbb, 0xdc, 0x7f, 0x50, 0x49, 0x33, 0x4c, 0xf1, 0x12, 0x13, 0x94, 0x5d, 0x57,
      0xe5, 0xac, 0x7d, 0x05, 0x5d, 0x04, 0x2b, 0x7e, 0x02, 0x4a, 0xa2, 0xb2, 0xf0, 0x8f, 0x0a, 0x91, 0x26, 0x08, 0x05, 0x27,
      0x2d, 0xc5, 0x10, 0x51, 0xc6, 0xe4, 0x7a, 0xd4, 0xfa, 0x40, 0x3b, 0x02, 0xb4, 0x51, 0x0b, 0x64, 0x7a, 0xe3, 0xd1, 0x77,
      0x0b, 0xac, 0x03, 0x26, 0xa8, 0x05, 0xbb, 0xef, 0xd4, 0x80, 0x56, 0xc8, 0xc1, 0x21, 0xbd, 0xb8};
  G2Affine g;
  g2_decode(gen, &g);
  const Fr hs = h_scalar.from_mont(), xs = x.from_mont();
  const G2Affine h = g2_to_affine(g2_mul(g, hs.v));
  g2_encode(h, out);
  g2_encode(g2_to_affine(g2_mul(h, xs.v)), out + 96);
}

// e(P_k, Q_k) as an Fp12 (tests only); an identity on either side gives 1.
__global__ void k_pairing_selftest(const uint4* g1, const LineCoeffs* lines, const int* ok, size_t n, uint32_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p[2] = {ld_aff(g1 + 6 * i), {Fp::zero(), Fp::zero()}};
  if (ok[i] != 1) p[0] = p[1];
  const LineCoeffs* l[2] = {lines + (size_t)PB_G2_LINES * i, lines};
  const Fp12 f = final_exponentiation(miller_loop2(p, l));
  const Fp* c = &f.c0.c0.c0;
  for (int k = 0; k < 12; k++)
    for (int j = 0; j < 12; j++) out[(i * 12 + k) * 12 + j] = c[k].v[j];
}

// ---- host side ------------------------------------------------------------------------------------------------
std::once_flag g_consts_once;
int g_consts_rc = 0;
int upload_pairing_consts() {
  std::call_once(g_consts_once, [] {
    pairing_consts_init();
    g_consts_rc = cudaMemcpyToSymbol(c_pairing, &h_pairing, sizeof h_pairing) == cudaSuccess ? 0 : 1;
  });
  return g_consts_rc ? fail(PB200_ERR_CUDA, "uploading the Frobenius coefficients") : 0;
}

// Decodes and prepares G2 points on the device: ok as k_g2_prepare, lines to d_lines (device).
int g2_prepare_dev(const uint8_t* enc, int count, LineCoeffs* d_lines, int* ok, cudaStream_t st) {
  PB_TRY(upload_pairing_consts());
  uint8_t* d_enc = nullptr;
  int* d_ok = nullptr;
  PB_CUDA(cudaMallocAsync((void**)&d_enc, 96 * (size_t)count, st));
  cudaError_t e = cudaMallocAsync((void**)&d_ok, sizeof(int) * count, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_enc, enc, 96 * (size_t)count, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    PB_LAUNCH(k_g2_prepare, div_up(count, 32), 32, 0, st, d_enc, count, d_lines, d_ok);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(ok, d_ok, sizeof(int) * count, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFreeAsync(d_enc, st);
  if (d_ok) cudaFreeAsync(d_ok, st);
  PB_CUDA(e);
  return 0;
}

// OpeningKey::from_bytes (key.rs:609-648): g, h and [x]h decoded with the on-curve and subgroup checks, the identity
// refused (OpeningKey::try_new).  g_raw (96 bytes) receives g when given; d_lines, when given, the prepared lines of
// [x]h then h.
int opening_key_decode(const uint8_t* opening_key, uint8_t* g_raw, LineCoeffs* d_lines) {
  uint8_t raw[96];
  PB_TRY(g1_decompress(opening_key, 1, 1, raw));
  bool g_inf = true;
  for (int k = 0; k < 96; k++) g_inf = g_inf && raw[k] == 0;
  uint8_t g2[2 * 96];
  memcpy(g2, opening_key + 48 + 96, 96);  // [x]H first: the pair of -(W_z + u W_zw)
  memcpy(g2 + 96, opening_key + 48, 96);
  int ok[2] = {0, 0};
  PB_TRY(g2_prepare_dev(g2, 2, d_lines, ok, thread_stream()));
  if (g_inf || ok[0] != 1 || ok[1] != 1)
    return fail(PB200_ERR_POINT_MALFORMED, "InvalidData: opening key point is the identity, not on the curve or not in the subgroup");
  if (g_raw) memcpy(g_raw, raw, 96);
  return 0;
}

uint64_t be64(const uint8_t* b) {
  uint64_t x = 0;
  for (int k = 0; k < 8; k++) x = (x << 8) | b[k];
  return x;
}
void put_be64(std::vector<uint8_t>& o, uint64_t x) {
  for (int k = 7; k >= 0; k--) o.push_back((uint8_t)(x >> (8 * k)));
}

// VerifierKey::to_bytes (widget.rs:84-111): VerifierKey::n, the 15 commitments in kKeyFileOrder, then 5 more
constexpr size_t kVerifierKeyBytes = 20 * 48 + 8;

// Verifier::new (verifier.rs:32-60) from validated parts.  vk_n is VerifierKey::n, which Compiler::compile sets to the
// constraint count (compiler.rs:278-279); the domain is EvaluationDomain::new(vk_n).
int verifier_build(const uint8_t* label, size_t label_len, uint64_t vk_n, uint64_t size, uint64_t constraints, const uint8_t* comms,
                   const uint8_t* opening_key, const uint64_t* pi_idx, size_t n_pi, pb200_verifier** out) {
  PB_TRY(ensure_init());
  // the 15 commitments: checked decoding (Commitment / G1Affine::from_bytes); then the opening key, with its lines
  std::vector<uint8_t> raw(16 * 96);
  PB_TRY(g1_decompress(comms, 15, 1, raw.data()));
  LineCoeffs* d_lines = nullptr;
  PB_CUDA(cudaMalloc((void**)&d_lines, 2 * PB_G2_LINES * sizeof(LineCoeffs)));
  int rc = opening_key_decode(opening_key, raw.data() + 15 * 96, d_lines);
  // EvaluationDomain::new (domain.rs:118-160)
  int log_n = 0;
  while (rc == 0 && log_n < 64 && ((uint64_t)1 << log_n) < vk_n) log_n++;
  if (rc == 0 && log_n >= 32) rc = fail(PB200_ERR_INVALID_DOMAIN, "InvalidEvalDomainSize");
  if (rc) {
    cudaFree(d_lines);
    return rc;
  }
  pb200_verifier* V = new pb200_verifier();
  V->d_lines = d_lines;
  V->label.assign(label, label + label_len);
  V->vk_n = vk_n;
  V->size = size;
  V->constraints = constraints;
  memcpy(V->vk_comm, comms, 15 * 48);
  memcpy(V->opening_key, opening_key, PB200_OPENING_KEY_BYTES);
  V->pi_idx.assign(pi_idx, pi_idx + n_pi);
  // ROOT_OF_UNITY = 7^((r - 1) / 2^32), squared down to the domain
  uint64_t t[4];
  memcpy(t, pbh::kFrMod.p, 32);
  t[0] -= 1;
  for (int k = 0; k < 4; k++) t[k] = (t[k] >> 32) | (k < 3 ? t[k + 1] << 32 : 0);
  HFr g = HFr::from_u64(7).pow(t, 4);
  for (int k = log_n; k < 32; k++) g = g.sqr();
  VerifyKeyHost& K = V->key;
  K.n = (uint64_t)1 << log_n;
  K.group_gen = g;
  K.size_fr = HFr::from_u64(K.n);
  K.size_inv = K.size_fr.inv();
  const HFr g_inv = g.inv();
  for (uint64_t idx : V->pi_idx) K.pi_roots.push_back(g_inv.pow_u64(idx));
  // Verifier::transcript (Transcript::base, V1 and V2) and Transcript::base_v3 (V3): built once for every version
  K.base_v3 = pbh::seed_transcript(V->label.data(), V->label.size(), constraints, comms, vk_n);
  K.base_legacy = pbh::seed_transcript_legacy(V->label.data(), V->label.size(), constraints, comms, vk_n);
  cudaError_t e = cudaMalloc((void**)&V->d_points, 16 * 96);
  if (e == cudaSuccess) e = cudaMemcpy(V->d_points, raw.data(), 16 * 96, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(V->d_points);
    cudaFree(V->d_lines);
    delete V;
    return fail(PB200_ERR_CUDA, "verifier key upload", cudaGetErrorString(e));
  }
  *out = V;
  return 0;
}

// Proofs [first, first + n) of a replay: checked under V and version, proof j of the group at proofs + 1008 j with
// its V->pi_idx.size() public inputs at pi_vals + 4 n_pi j.
struct ReplayGroup {
  const pb200_verifier* V;
  int version;
  const uint8_t* proofs;
  const uint64_t* pi_vals;
  size_t first, n;
};

// The host stage of pb200_verify_with_version and batch verification, over every group's proofs at once (groups in
// order, covering [0, n_proofs)): per proof its commitments (comm), the 32 scalars of k_verify_msm (scal), the host's
// verdict (hstat) and, when us is given, its challenge u; spread over threads for large calls.
void replay(const std::vector<ReplayGroup>& groups, size_t n_proofs, std::vector<uint64_t>& scal, std::vector<int>& hstat,
            std::vector<uint8_t>& comm, HFr* us) {
  scal.assign(n_proofs * PB_VERIFY_TERMS * 4, 0);
  hstat.assign(n_proofs, 0);
  comm.assign(n_proofs * kProofEvalAt, 0);
  auto work = [&](size_t lo, size_t hi) {
    size_t g = 0;
    for (size_t i = lo; i < hi; i++) {
      while (i >= groups[g].first + groups[g].n) g++;
      const ReplayGroup& G = groups[g];
      const size_t j = i - G.first, n_pi = G.V->pi_idx.size();
      const uint8_t* pr = G.proofs + kProofBytes * j;
      memcpy(comm.data() + kProofEvalAt * i, pr, kProofEvalAt);
      hstat[i] = verify_scalars(G.V->key, G.version, pr, (const HFr*)(G.pi_vals + 4 * n_pi * j), scal.data() + (size_t)PB_VERIFY_TERMS * 4 * i,
                                us ? us + i : nullptr);
    }
  };
  const size_t n_thr = std::min<size_t>(std::max(1u, std::thread::hardware_concurrency()), std::min<size_t>(16, (n_proofs + 31) / 32));
  if (n_thr <= 1) {
    work(0, n_proofs);
  } else {
    std::vector<std::thread> th;
    const size_t per = (n_proofs + n_thr - 1) / n_thr;
    for (size_t t = 0; t < n_thr; t++) th.emplace_back(work, std::min(n_proofs, t * per), std::min(n_proofs, (t + 1) * per));
    for (auto& x : th) x.join();
  }
}

// pb200_batch_verify_groups (pb200_batch_verify is its one-group case); points, when given, receives sum w_i L_i then
// sum w_i R_i (96-byte raw affine each; zeros when the verdict is decided before the pairing).
int batch_verify(const pb200_verifier_t* const* Vs, const int32_t* versions, const size_t* n_proofs, const size_t* n_pi, size_t n_groups,
                 const uint8_t* proofs, const uint64_t* pi_vals, int32_t* verdict, uint8_t* points) {
  PB_TRY(ensure_init());
  if (!verdict || (n_groups && (!Vs || !versions || !n_proofs || !n_pi))) return fail(PB200_ERR_INVALID_ARG, "null argument");
  // the groups in call order, and one key slot per distinct verifier (slots in order of first appearance)
  std::vector<ReplayGroup> groups(n_groups);
  std::vector<const pb200_verifier*> slot_v;
  std::unordered_map<const pb200_verifier*, uint32_t> slot_index;
  std::vector<uint32_t> slot_of(n_groups);
  size_t n = 0, n_pi_words = 0;
  for (size_t g = 0; g < n_groups; g++) {
    const pb200_verifier* V = Vs[g];
    if (!V) return fail(PB200_ERR_INVALID_ARG, "null argument");
    if (versions[g] != PB200_PLONK_V1 && versions[g] != PB200_PLONK_V2 && versions[g] != PB200_PLONK_V3)
      return fail(PB200_ERR_INVALID_ARG, "unknown PlonkVersion");
    if (n_pi[g] != V->pi_idx.size()) return fail(PB200_ERR_INVALID_ARG, "InconsistentPublicInputsLen");
    if (memcmp(V->opening_key, Vs[0]->opening_key, PB200_OPENING_KEY_BYTES))
      return fail(PB200_ERR_INVALID_ARG, "the verifiers of one batch must share one opening key (one SRS)");
    const auto slot = slot_index.emplace(V, (uint32_t)slot_v.size());
    if (slot.second) slot_v.push_back(V);
    slot_of[g] = slot.first->second;
    n += n_proofs[g];
    n_pi_words += 4 * n_pi[g] * n_proofs[g];
  }
  if ((!proofs && n) || (!pi_vals && n_pi_words)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  for (size_t g = 0, first = 0, pi_at = 0; g < n_groups; g++) {
    groups[g] = {Vs[g], versions[g], proofs ? proofs + kProofBytes * first : nullptr, pi_vals ? pi_vals + pi_at : nullptr, first, n_proofs[g]};
    first += n_proofs[g];
    pi_at += 4 * n_pi[g] * n_proofs[g];
  }
  if (points) memset(points, 0, 2 * 96);
  if (!n) {  // batch_check rejects an empty batch (key.rs:667-669)
    *verdict = PB200_ERR_VERIFY;
    return 0;
  }
  PB_TRY(upload_pairing_consts());
  std::vector<uint64_t> scal;
  std::vector<int> hstat;
  std::vector<uint8_t> comm;
  std::vector<HFr> us(n);
  replay(groups, n, scal, hstat, comm, us.data());
  bool host_ok = true;
  for (int h : hstat) {
    if (h == PB200_ERR_POINT_MALFORMED) {
      *verdict = PB200_ERR_POINT_MALFORMED;
      return 0;
    }
    host_ok = host_ok && h == PB200_OK;
  }
  // rho is needed only when every proof passed the host stage; otherwise the verdict is a failure whatever the
  // weights, and the device still looks for malformed commitments, which take precedence
  const std::vector<HFr> w = host_ok ? batch_weights(batch_challenge(versions, n_proofs, n_groups, us.data()), n) : std::vector<HFr>(n, HFr::zero());
  // k_batch_fold's blocks slot by slot: each group's proofs in runs of kBatchFoldWarps, so no block spans two slots
  // (one group gives blocks {8 b, min(8, n - 8 b)}); slot_blocks[s] is slot s's first block
  const size_t n_slots = slot_v.size();
  std::vector<size_t> order(n_groups);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return slot_of[a] < slot_of[b]; });
  std::vector<FoldBlock> blocks;
  std::vector<uint32_t> slot_blocks(n_slots + 1, 0);
  for (size_t g : order) {
    for (size_t j = 0; j < n_proofs[g]; j += kBatchFoldWarps)
      blocks.push_back({(uint32_t)(groups[g].first + j), (uint32_t)std::min<size_t>(kBatchFoldWarps, n_proofs[g] - j)});
    slot_blocks[slot_of[g] + 1] = (uint32_t)blocks.size();
  }
  const size_t fold_blocks = blocks.size();
  const size_t n_r = 11 * n + 16 * n_slots, r_pad = (n_r + 31) / 32 * 32, n_l = 2 * n, l_pad = (n_l + 31) / 32 * 32;
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint8_t* d_comm;
  uint4 *d_pts, *d_scal, *d_w, *d_rs, *d_ls, *d_keypart, *d_keypts, *d_g1;
  FoldBlock* d_blocks;
  uint32_t* d_slot_blocks;
  G1Xyzz* d_part;
  unsigned *d_bad, *d_flags;
  int *d_stat, *d_verdict;
  PB_ALLOC(scope, d_comm, n * kProofEvalAt);
  PB_ALLOC(scope, d_pts, n * 11 * 96);
  PB_ALLOC(scope, d_scal, scal.size() * 8);
  PB_ALLOC(scope, d_w, n * 32);
  PB_ALLOC(scope, d_rs, n_r * 32);
  PB_ALLOC(scope, d_ls, n_l * 32);
  PB_ALLOC(scope, d_keypart, fold_blocks * 16 * 32);
  PB_ALLOC(scope, d_keypts, n_slots * 16 * 96);
  PB_ALLOC(scope, d_blocks, fold_blocks * sizeof(FoldBlock));
  PB_ALLOC(scope, d_slot_blocks, slot_blocks.size() * sizeof(uint32_t));
  PB_ALLOC(scope, d_part, (r_pad + l_pad) / 32 * sizeof(G1Xyzz));
  PB_ALLOC(scope, d_g1, 2 * 96);
  PB_ALLOC(scope, d_bad, 4);
  PB_ALLOC(scope, d_flags, 4);
  PB_ALLOC(scope, d_stat, n * sizeof(int));
  PB_ALLOC(scope, d_verdict, sizeof(int));
  static_assert(sizeof(HFr) == 32, "HFr: four little-endian words, the layout of a device Fr");
  PB_CUDA(cudaMemcpyAsync(d_comm, comm.data(), n * kProofEvalAt, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_scal, scal.data(), scal.size() * 8, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_w, w.data(), n * 32, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_stat, hstat.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_blocks, blocks.data(), fold_blocks * sizeof(FoldBlock), cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_slot_blocks, slot_blocks.data(), slot_blocks.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  for (size_t s = 0; s < n_slots; s++)  // each slot's 16 key points: the 15 commitments, then opening_key.g
    PB_CUDA(cudaMemcpyAsync(d_keypts + 16 * 6 * s, slot_v[s]->d_points, 16 * 96, cudaMemcpyDeviceToDevice, st));
  PB_CUDA(cudaMemsetAsync(d_flags, 0, 4, st));
  PB_CUDA(cudaMemsetAsync(d_g1, 0, 2 * 96, st));
  g1_decompress_dev(d_comm, n * 11, d_pts, d_bad, st);
  PB_LAUNCH(k_batch_fold, fold_blocks, 32 * kBatchFoldWarps, 0, st, d_pts, d_comm, d_scal, d_w, d_stat, d_blocks, d_flags, d_rs, d_ls, d_keypart);
  PB_LAUNCH(k_batch_key_sums, 16 * n_slots, 256, 0, st, d_keypart, d_slot_blocks, d_flags, d_verdict, d_rs + 2 * 11 * n);
  PB_LAUNCH(k_batch_msm, div_up(r_pad + l_pad, 128), 128, 0, st, d_keypts, d_pts, d_rs, 11 * n, n_r, r_pad, d_ls, n_l, l_pad, d_verdict,
            d_part);
  PB_LAUNCH(k_batch_reduce, 2, 256, 0, st, d_part, r_pad / 32, l_pad / 32, d_verdict, d_g1);
  // the verifiers share their opening key, so the first one's prepared [x]H and H serve the whole call
  PB_LAUNCH(k_verify_pairing, 1, 64, 0, st, d_g1, Vs[0]->d_lines, 1, d_verdict);
  PB_CUDA(cudaGetLastError());
  int v = 0;
  PB_CUDA(cudaMemcpyAsync(&v, d_verdict, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (points) PB_CUDA(cudaMemcpyAsync(points, d_g1, 2 * 96, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  *verdict = v;
  return 0;
}

}  // namespace

int opening_key_check(const uint8_t* opening_key) { return opening_key_decode(opening_key, nullptr, nullptr); }

int opening_key_g2(const uint64_t* x_mont, const uint64_t* h_scalar_mont, uint8_t* out_2x96) {
  cudaStream_t st = thread_stream();
  Fr x, hs;
  memcpy(x.v, x_mont, 32);
  memcpy(hs.v, h_scalar_mont, 32);
  uint8_t* d_out = nullptr;
  PB_CUDA(cudaMallocAsync((void**)&d_out, 2 * 96, st));
  PB_LAUNCH(k_opening_key_g2, 1, 32, 0, st, x, hs, d_out);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_2x96, d_out, 2 * 96, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFreeAsync(d_out, st);
  PB_CUDA(e);
  return 0;
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb200_verifier_new(const uint8_t* label, size_t label_len, size_t n_constraints, const uint8_t* vk_comms_15x48,
                       const uint8_t* opening_key, const uint64_t* pi_idx, size_t n_pi, pb200_verifier_t** out) {
  if ((!label && label_len) || !vk_comms_15x48 || !opening_key || (!pi_idx && n_pi) || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  uint64_t size = 1;  // Verifier::size = constraints.next_power_of_two() (compiler.rs:141)
  while (size < n_constraints && size) size <<= 1;
  if (!size) return fail(PB200_ERR_INVALID_DOMAIN, "InvalidEvalDomainSize");
  return verifier_build(label, label_len, n_constraints, size, n_constraints, vk_comms_15x48, opening_key, pi_idx, n_pi, out);
}

int pb200_verifier_from_bytes(const uint8_t* bytes, size_t len, pb200_verifier_t** out) {
  if (!bytes || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (len < 48) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes");
  const uint64_t label_len = be64(bytes), vk_len = be64(bytes + 8), ok_len = be64(bytes + 16), n_pi = be64(bytes + 24);
  const uint64_t size = be64(bytes + 32), constraints = be64(bytes + 40);
  // checked arithmetic as verifier.rs:150-165: any overflow is NotEnoughBytes
  if (n_pi > UINT64_MAX / 8) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes");
  uint64_t need = label_len;
  for (uint64_t add : {vk_len, ok_len, n_pi * 8}) {
    if (need > UINT64_MAX - add) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes");
    need += add;
  }
  if (len - 48 < need) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes");
  const uint8_t* p = bytes + 48;
  const uint8_t* label = p;
  const uint8_t* vk = label + label_len;
  const uint8_t* okey = vk + vk_len;
  const uint8_t* pis = okey + ok_len;
  // VerifierKey::from_slice / OpeningKey::from_slice read exactly their sizes
  if (vk_len < kVerifierKeyBytes || ok_len < PB200_OPENING_KEY_BYTES) return fail(PB200_ERR_INVALID_ARG, "BadLength");
  uint64_t n = 0;
  for (int k = 7; k >= 0; k--) n = (n << 8) | vk[k];
  uint8_t comms[15 * 48];
  for (int k = 0; k < 15; k++) memcpy(comms + 48 * k, vk + 8 + 48 * k, 48);
  uint8_t ordered[15 * 48];
  for (int k = 0; k < 15; k++) memcpy(ordered + 48 * kKeyFileOrder[k], comms + 48 * k, 48);
  std::vector<uint64_t> idx(n_pi);
  for (uint64_t k = 0; k < n_pi; k++) idx[k] = be64(pis + 8 * k);
  return verifier_build(label, label_len, n, size, constraints, ordered, okey, idx.data(), idx.size(), out);
}

int pb200_verifier_to_bytes(const pb200_verifier_t* V, uint8_t* out, size_t cap, size_t* len) {
  if (!V || !len) return fail(PB200_ERR_INVALID_ARG, "null argument");
  std::vector<uint8_t> o;
  put_be64(o, V->label.size());
  put_be64(o, kVerifierKeyBytes);
  put_be64(o, PB200_OPENING_KEY_BYTES);
  put_be64(o, V->pi_idx.size());
  put_be64(o, V->size);
  put_be64(o, V->constraints);
  o.insert(o.end(), V->label.begin(), V->label.end());
  const size_t vk_at = o.size();
  for (int k = 0; k < 8; k++) o.push_back((uint8_t)(V->vk_n >> (8 * k)));
  for (int k = 0; k < 15; k++) o.insert(o.end(), V->vk_comm[kKeyFileOrder[k]], V->vk_comm[kKeyFileOrder[k]] + 48);
  o.resize(vk_at + kVerifierKeyBytes, 0);
  o.insert(o.end(), V->opening_key, V->opening_key + PB200_OPENING_KEY_BYTES);
  for (uint64_t i : V->pi_idx) put_be64(o, i);
  *len = o.size();
  if (!out) return 0;
  if (cap < o.size()) return fail(PB200_ERR_INVALID_ARG, "output buffer too small");
  memcpy(out, o.data(), o.size());
  return 0;
}

void pb200_verifier_free(pb200_verifier_t* V) {
  if (!V) return;
  ensure_init();
  cudaFree(V->d_points);
  cudaFree(V->d_lines);
  delete V;
}

int pb200_verify(const pb200_verifier_t* V, const uint8_t* proofs, size_t n_proofs, const uint64_t* pi_vals, size_t n_pi,
                 int32_t* status) {
  return pb200_verify_with_version(V, PB200_PLONK_V3, proofs, n_proofs, pi_vals, n_pi, status);
}

int pb200_verify_with_version(const pb200_verifier_t* V, int version, const uint8_t* proofs, size_t n_proofs,
                              const uint64_t* pi_vals, size_t n_pi, int32_t* status) {
  PB_TRY(ensure_init());
  if (!V || (!proofs && n_proofs) || (!pi_vals && n_pi && n_proofs) || (!status && n_proofs)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (version != PB200_PLONK_V1 && version != PB200_PLONK_V2 && version != PB200_PLONK_V3)
    return fail(PB200_ERR_INVALID_ARG, "unknown PlonkVersion");
  if (n_pi != V->pi_idx.size()) return fail(PB200_ERR_INVALID_ARG, "InconsistentPublicInputsLen");
  if (!n_proofs) return 0;
  PB_TRY(upload_pairing_consts());
  std::vector<uint64_t> scal;
  std::vector<int> hstat;
  std::vector<uint8_t> comm;
  replay({{V, version, proofs, pi_vals, 0, n_proofs}}, n_proofs, scal, hstat, comm, nullptr);
  // device: decoding, the two G1 points, the pairing check
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint8_t* d_comm;
  uint4 *d_pts, *d_scal, *d_g1;
  unsigned* d_bad;
  int* d_stat;
  PB_ALLOC(scope, d_comm, n_proofs * kProofEvalAt);
  PB_ALLOC(scope, d_pts, n_proofs * 11 * 96);
  PB_ALLOC(scope, d_scal, scal.size() * 8);
  PB_ALLOC(scope, d_g1, n_proofs * 2 * 96);
  PB_ALLOC(scope, d_bad, 4);
  PB_ALLOC(scope, d_stat, n_proofs * sizeof(int));
  PB_CUDA(cudaMemcpyAsync(d_comm, comm.data(), n_proofs * kProofEvalAt, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_scal, scal.data(), scal.size() * 8, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_stat, hstat.data(), n_proofs * sizeof(int), cudaMemcpyHostToDevice, st));
  g1_decompress_dev(d_comm, n_proofs * 11, d_pts, d_bad, st);
  PB_LAUNCH(k_verify_msm, div_up(n_proofs * 32, 128), 128, 0, st, V->d_points, d_pts, d_comm, d_scal, n_proofs, d_stat, d_g1);
  PB_LAUNCH(k_verify_pairing, div_up(n_proofs, 64), 64, 0, st, d_g1, V->d_lines, n_proofs, d_stat);
  PB_CUDA(cudaGetLastError());
  PB_CUDA(cudaMemcpyAsync(hstat.data(), d_stat, n_proofs * sizeof(int), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < n_proofs; i++) status[i] = hstat[i];
  return 0;
}

int pb200_batch_verify(const pb200_verifier_t* V, int version, const uint8_t* proofs, size_t n_proofs, const uint64_t* pi_vals,
                       size_t n_pi, int32_t* verdict) {
  return batch_verify(&V, &version, &n_proofs, &n_pi, 1, proofs, pi_vals, verdict, nullptr);
}

int pb200_selftest_batch_verify_points(const pb200_verifier_t* V, int version, const uint8_t* proofs, size_t n_proofs,
                                       const uint64_t* pi_vals, size_t n_pi, int32_t* verdict, uint8_t* points_2x96) {
  if (!points_2x96) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return batch_verify(&V, &version, &n_proofs, &n_pi, 1, proofs, pi_vals, verdict, points_2x96);
}

int pb200_batch_verify_groups(const pb200_verifier_t* const* verifiers, const int32_t* versions, const size_t* n_proofs,
                              const size_t* n_pi, size_t n_groups, const uint8_t* proofs, const uint64_t* pi_vals, int32_t* verdict) {
  return batch_verify(verifiers, versions, n_proofs, n_pi, n_groups, proofs, pi_vals, verdict, nullptr);
}

int pb200_selftest_batch_verify_groups_points(const pb200_verifier_t* const* verifiers, const int32_t* versions, const size_t* n_proofs,
                                              const size_t* n_pi, size_t n_groups, const uint8_t* proofs, const uint64_t* pi_vals,
                                              int32_t* verdict, uint8_t* points_2x96) {
  if (!points_2x96) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return batch_verify(verifiers, versions, n_proofs, n_pi, n_groups, proofs, pi_vals, verdict, points_2x96);
}

int pb200_selftest_pairing(const uint64_t* g1_raw, const uint8_t* g2_compressed, size_t n, uint64_t* out_fp12) {
  PB_TRY(ensure_init());
  if (!n) return 0;
  if (!g1_raw || !g2_compressed || !out_fp12) return fail(PB200_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  LineCoeffs* d_lines;
  uint4* d_g1;
  int* d_ok;
  uint32_t* d_out;
  PB_ALLOC(scope, d_lines, n * PB_G2_LINES * sizeof(LineCoeffs));
  PB_ALLOC(scope, d_g1, n * 96);
  PB_ALLOC(scope, d_ok, n * sizeof(int));
  PB_ALLOC(scope, d_out, n * 576);
  std::vector<int> ok(n);
  PB_TRY(g2_prepare_dev(g2_compressed, (int)n, d_lines, ok.data(), st));
  for (size_t i = 0; i < n; i++)
    if (!ok[i]) return fail(PB200_ERR_POINT_MALFORMED, "malformed G2 encoding");
  PB_CUDA(cudaMemcpyAsync(d_ok, ok.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_g1, g1_raw, n * 96, cudaMemcpyHostToDevice, st));
  PB_LAUNCH(k_pairing_selftest, div_up(n, 32), 32, 0, st, d_g1, d_lines, d_ok, n, d_out);
  PB_CUDA(cudaGetLastError());
  PB_CUDA(cudaMemcpyAsync(out_fp12, d_out, n * 576, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  return 0;
}
}
