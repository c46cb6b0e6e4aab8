// Lagrange form of a commit key on the GPU: inverse NTT over G1 points (csrc/ecntt.cuh).
//
// prover_build (prover.cu) makes the Lagrange-form key of the wire commitments with it; it is also
// exposed as pb200_g1_lagrange_key so that the transform can be checked on its own.  One thread per
// butterfly, log n launches; a butterfly is one XYZZ addition, one subtraction and a 255-bit
// double-and-add (~380 group operations), so the whole transform is ~n/2 log n * 380 group
// operations - about 2e8 at n = 2^16 - once per key.
#include "internal.cuh"
#include "ecntt.cuh"

namespace pb {
namespace {

PB_D Fp ec_ld_fp(const uint4* q) {
  const uint4 a = q[0], b = q[1], c = q[2];
  Fp f;
  f.v[0] = a.x; f.v[1] = a.y; f.v[2] = a.z; f.v[3] = a.w;
  f.v[4] = b.x; f.v[5] = b.y; f.v[6] = b.z; f.v[7] = b.w;
  f.v[8] = c.x; f.v[9] = c.y; f.v[10] = c.z; f.v[11] = c.w;
  return f;
}
PB_D void ec_st_fp(uint4* q, const Fp& f) {
  q[0] = make_uint4(f.v[0], f.v[1], f.v[2], f.v[3]);
  q[1] = make_uint4(f.v[4], f.v[5], f.v[6], f.v[7]);
  q[2] = make_uint4(f.v[8], f.v[9], f.v[10], f.v[11]);
}
PB_D G1Xyzz ec_ld_xyzz(const uint4* p, size_t i) {
  G1Xyzz a;
  a.x = FpR::from(ec_ld_fp(p + 12 * i));
  a.y = FpR::from(ec_ld_fp(p + 12 * i + 3));
  a.zz = FpR::from(ec_ld_fp(p + 12 * i + 6));
  a.zzz = FpR::from(ec_ld_fp(p + 12 * i + 9));
  return a;
}
PB_D void ec_st_xyzz(uint4* p, size_t i, const G1Xyzz& a) {  // canonical, like every stored XYZZ point
  const G1Xyzz c = a.canonical();
  ec_st_fp(p + 12 * i, c.x.raw());
  ec_st_fp(p + 12 * i + 3, c.y.raw());
  ec_st_fp(p + 12 * i + 6, c.zz.raw());
  ec_st_fp(p + 12 * i + 9, c.zzz.raw());
}
PB_D Fr ec_ld_fr(const uint4* p, size_t i) {
  const uint4 a = p[2 * i], b = p[2 * i + 1];
  Fr f;
  f.v[0] = a.x; f.v[1] = a.y; f.v[2] = a.z; f.v[3] = a.w;
  f.v[4] = b.x; f.v[5] = b.y; f.v[6] = b.z; f.v[7] = b.w;
  return f;
}

// affine (96 B, identity = zeros) -> XYZZ
__global__ void k_ec_load(const uint4* aff, size_t n, uint4* A) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p;
  p.x = ec_ld_fp(aff + 6 * i);
  p.y = ec_ld_fp(aff + 6 * i + 3);
  ec_st_xyzz(A, i, G1Xyzz::from_affine(p));
}

// stage s of the decimation-in-frequency transform: blocks of len = n >> s, butterfly (j, j + len/2)
// with twiddle w_n^(-(j << s)); tw[k] = w_n^(-k), k < n/2
__global__ void __launch_bounds__(128) k_ec_stage(uint4* A, size_t n, int s, const uint4* tw) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n / 2) return;
  const size_t len = n >> s, half = len >> 1;
  const size_t blk = t / half, j = t % half, i0 = blk * len + j, ex = j << s;
  G1Xyzz a = ec_ld_xyzz(A, i0), b = ec_ld_xyzz(A, i0 + half);
  ec_butterfly(a, b, ec_ld_fr(tw, ex), ex == 0);
  ec_st_xyzz(A, i0, a);
  ec_st_xyzz(A, i0 + half, b);
}

struct EcScalar {
  uint32_t k[8];
};
// out[bitrev(i)] = affine(A[i] / n)
__global__ void __launch_bounds__(128) k_ec_finish(const uint4* A, size_t n, int log_n, EcScalar n_inv, uint4* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const G1Affine r = xyzz_to_affine(xyzz_mul(ec_ld_xyzz(A, i), n_inv.k, 8));
  const size_t o = ec_bitrev((unsigned)i, log_n);
  ec_st_fp(out + 6 * o, r.x);
  ec_st_fp(out + 6 * o + 3, r.y);
}

}  // namespace

// d_in, d_out: n = 2^log_n affine points (96 B each) on the device; d_out may not alias d_in.
int lagrange_key_dev(const uint4* d_in, int log_n, uint4* d_out, cudaStream_t st) {
  if (log_n < 0 || log_n > 28) return fail(PB200_ERR_INVALID_DOMAIN, "group-element NTT size");
  const size_t n = (size_t)1 << log_n;
  uint4* A = nullptr;
  PB_CUDA(cudaMalloc((void**)&A, n * 192));
  struct Free {
    uint4* p;
    ~Free() { cudaFree(p); }
  } guard{A};
  PB_LAUNCH(k_ec_load, div_up(n, 128), 128, 0, st, d_in, n, A);
  if (log_n > 0) {
    const uint4* tw = nullptr;
    PB_TRY(get_twiddles(log_n, true, st, &tw));
    for (int s = 0; s < log_n; s++) PB_LAUNCH(k_ec_stage, div_up(n / 2, 128), 128, 0, st, A, n, s, tw);
  }
  EcScalar ninv;
  const Fr c = ntt_size_inv(log_n).from_mont();
  for (int i = 0; i < 8; i++) ninv.k[i] = c.v[i];
  PB_LAUNCH(k_ec_finish, div_up(n, 128), 128, 0, st, (const uint4*)A, n, log_n, ninv, d_out);
  PB_CUDA(cudaGetLastError());
  PB_CUDA(stream_wait(st));
  return 0;
}

}  // namespace pb
