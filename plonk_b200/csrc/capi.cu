// extern "C" surface of libplonk_b200 (see include/plonk_b200.h for the reference call sites each
// entry point replaces).  Host-pointer variants stage through stream-ordered device allocations;
// there is no CPU fallback anywhere: without a usable CUDA device every call returns PB200_ERR_CUDA.
#include <dlfcn.h>

#include <mutex>
#include <vector>

#include "internal.cuh"
#include "host_field.h"

namespace pb {
thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

std::atomic<unsigned> g_num_sms{0};

static std::mutex g_init_mu;
static int g_device = -1;

// Binds the process to `dev` (with g_init_mu held): the device every later call uses, and its SM count.
static int bind_device(int dev) {
  int sms = 0;
  PB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  g_num_sms.store((unsigned)sms, std::memory_order_relaxed);
  g_device = dev;
  return 0;
}

// Per-call workspaces come from the stream-ordered pool; keep freed blocks cached instead of
// returning them to the driver at every synchronisation.
static void keep_pool(int device) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
}

int ensure_init() {
  std::lock_guard<std::mutex> lk(g_init_mu);
  if (g_device >= 0) {
    PB_CUDA(cudaSetDevice(g_device));
    return 0;
  }
  int count = 0;
  PB_CUDA(cudaGetDeviceCount(&count));
  if (count == 0) return fail(PB200_ERR_CUDA, "no CUDA device");
  int dev = 0;
  PB_CUDA(cudaGetDevice(&dev));
  PB_TRY(bind_device(dev));
  keep_pool(dev);
  return 0;
}

cudaStream_t thread_stream() {
  static thread_local cudaStream_t st = nullptr;
  if (!st) {
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) st = nullptr;
  }
  return st;
}

cudaError_t stream_wait(cudaStream_t st) {
  static const bool spin = [] {
    const char* e = getenv("PB200_SPIN");
    return e && atoi(e) != 0;
  }();
  if (spin) return cudaStreamSynchronize(st);
  static thread_local cudaEvent_t ev = nullptr;
  if (!ev) {
    cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventBlockingSync | cudaEventDisableTiming);
    if (e != cudaSuccess) return e;
  }
  cudaError_t e = cudaEventRecord(ev, st);
  if (e != cudaSuccess) return e;
  return cudaEventSynchronize(ev);
}

void* pinned_scratch(size_t bytes, int slot) {
  static thread_local void* bufs[2] = {nullptr, nullptr};
  static thread_local size_t caps[2] = {0, 0};
  void*& buf = bufs[slot & 1];
  size_t& cap = caps[slot & 1];
  if (bytes > cap) {
    if (buf) cudaFreeHost(buf);
    buf = nullptr;
    cap = 0;
    const size_t want = bytes < (64u << 10) ? (64u << 10) : bytes;
    if (cudaHostAlloc(&buf, want, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    cap = want;
  }
  return buf;
}

// checked = 1: CommitKey::from_raw_var_bytes (key.rs:258-298: the length must be exact, zero points are an
// error); checked = 0: from_slice_unchecked (key.rs:242-256: as many whole records as the bytes hold, at most
// the announced count).  Writes the 96-byte layout when out_raw is given (identity -> zeros).
int raw_commit_key_parse(const uint8_t* bytes, size_t len, int checked, size_t* n_points, uint8_t* out_raw) {
  if (len < 8) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes: raw commit key shorter than its length prefix");
  uint64_t cnt = 0;
  for (int i = 7; i >= 0; i--) cnt = (cnt << 8) | bytes[i];
  const size_t have = (len - 8) / PB200_G1_RAW_SIZE;
  size_t n;
  if (checked) {
    if (cnt == 0) return fail(PB200_ERR_POINT_MALFORMED, "InvalidData: empty commit key");
    if (cnt > have || (len - 8) != (size_t)cnt * PB200_G1_RAW_SIZE) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes: raw commit key length does not match its point count");
    n = (size_t)cnt;
  } else {
    n = cnt < have ? (size_t)cnt : have;
  }
  *n_points = n;
  if (out_raw)
    for (size_t i = 0; i < n; i++) {
      const uint8_t* rec = bytes + 8 + i * PB200_G1_RAW_SIZE;
      if (rec[96])
        memset(out_raw + 96 * i, 0, 96);  // Choice(1): the identity, whatever its coordinates hold
      else
        memcpy(out_raw + 96 * i, rec, 96);
    }
  return 0;
}

// One record of CommitKey::to_raw_var_bytes (G1Affine::to_raw_bytes): the 96 raw bytes and a zero flag; this
// library's identity (96 zero bytes) becomes the reference's G1Affine::identity(): x = 0, y = 1 (Montgomery form),
// flag 1 - what raw_commit_key_parse maps back.
void raw_commit_key_record(const uint8_t* raw96, uint8_t* rec97) {
  bool zero = true;
  for (int i = 0; i < 96 && zero; i++) zero = raw96[i] == 0;
  memcpy(rec97, raw96, 96);
  if (zero) memcpy(rec97 + 48, pbh::kFpMod.r1, 48);
  rec97[96] = zero ? 1 : 0;
}

// A draw of util::random_nonzero_bls_scalar: a canonical Montgomery residue (below r) that is not zero.
static bool nonzero_canonical_scalar(const uint64_t* s) {
  if (!(s[0] | s[1] | s[2] | s[3])) return false;
  for (int k = 3; k >= 0; k--)
    if (s[k] != pbh::kFrMod.p[k]) return s[k] < pbh::kFrMod.p[k];
  return false;
}

int setup_args_check(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar) {
  if (!x || !g_scalar || !h_scalar) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (max_degree == 0) return fail(PB200_ERR_DEGREE_IS_ZERO, "DegreeIsZero");
  if (max_degree > SIZE_MAX / 96 - 7) return fail(PB200_ERR_INVALID_ARG, "max_degree too large");
  if (!nonzero_canonical_scalar(x) || !nonzero_canonical_scalar(g_scalar) || !nonzero_canonical_scalar(h_scalar))
    return fail(PB200_ERR_INVALID_ARG, "a setup draw is zero or not a canonical scalar");
  return 0;
}
}  // namespace pb

using namespace pb;

extern "C" {

int pb200_init(int device) {
  {
    std::lock_guard<std::mutex> lk(g_init_mu);
    int count = 0;
    PB_CUDA(cudaGetDeviceCount(&count));
    if (device < 0 || device >= count) return fail(PB200_ERR_CUDA, "no such CUDA device");
    // One device per process: twiddle/coset tables, per-thread streams and pinned buffers are created on
    // the first device used and are not keyed by device.
    if (g_device >= 0 && g_device != device)
      return fail(PB200_ERR_INVALID_ARG, "pb200_init: this process is already bound to another CUDA device (one device per process)");
    PB_CUDA(cudaSetDevice(device));
    if (g_device < 0) PB_TRY(bind_device(device));
  }
  keep_pool(device);
  return 0;
}

const char* pb200_last_error(void) { return g_last_error.c_str(); }

int pb200_device_sync(void) {
  PB_TRY(ensure_init());
  PB_CUDA(cudaDeviceSynchronize());
  return 0;
}

uint64_t pb200_launch_count(void) { return g_launches.load(); }

int pb200_ntt_dev(const uint64_t* d_in, size_t in_len, uint64_t* d_out, uint32_t log_n, int inverse, int coset,
                  uint32_t batch, size_t in_stride, size_t out_stride, void* stream) {
  PB_TRY(ensure_init());
  cudaStream_t st = stream ? (cudaStream_t)stream : thread_stream();
  return ntt_run(d_in, in_len, d_out, log_n, inverse, coset, batch, in_stride, out_stride, st, nullptr);
}

int pb200_ntt(const uint64_t* in, size_t in_len, uint64_t* out, uint32_t log_n, int inverse, int coset,
              uint32_t batch, size_t in_stride, size_t out_stride) {
  PB_TRY(ensure_init());
  if (log_n >= 32) return fail(PB200_ERR_INVALID_DOMAIN, "log_n >= TWO_ADACITY");
  if (batch == 0) return 0;
  if ((!in && in_len) || !out) return fail(PB200_ERR_INVALID_ARG, "null buffer");
  cudaStream_t st = thread_stream();
  const size_t n = (size_t)1 << log_n;
  const size_t use = in_len < n ? in_len : n;
  uint64_t *d_in = nullptr, *d_out = nullptr;
  PB_CUDA(cudaMallocAsync((void**)&d_out, (size_t)batch * n * 32, st));
  int rc = 0;
  if (use) {
    cudaError_t e = cudaMallocAsync((void**)&d_in, (size_t)batch * use * 32, st);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(d_in, use * 32, in, in_stride * 32, use * 32, batch, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) rc = fail(PB200_ERR_CUDA, "ntt input upload", cudaGetErrorString(e));
  }
  if (rc == 0) rc = ntt_run(d_in, use, d_out, log_n, inverse, coset, batch, use, n, st, nullptr);
  if (rc == 0) {
    cudaError_t e = cudaMemcpy2DAsync(out, out_stride * 32, d_out, n * 32, n * 32, batch, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = fail(PB200_ERR_CUDA, "ntt result copy", cudaGetErrorString(e));
  }
  if (d_in) cudaFreeAsync(d_in, st);
  cudaFreeAsync(d_out, st);
  return rc;
}

int pb200_srs_upload(const uint8_t* raw_points, size_t n_points, pb200_srs_t** out) {
  PB_TRY(ensure_init());
  if (!raw_points || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return srs_upload(raw_points, n_points, out, 0);
}
int pb200_srs_upload_window(const uint8_t* raw_points, size_t n_points, int window_bits, pb200_srs_t** out) {
  PB_TRY(ensure_init());
  if (!raw_points || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (window_bits != 0 && (window_bits < 2 || window_bits > 20)) return fail(PB200_ERR_INVALID_ARG, "window_bits must be 0 (automatic) or in 2..=20");
  return srs_upload(raw_points, n_points, out, window_bits);
}
int pb200_srs_window(const pb200_srs_t* srs) { return srs ? srs_window(srs) : 0; }
int pb200_msm_window_for(size_t n_points) { return msm_window_for(n_points); }
void pb200_srs_free(pb200_srs_t* srs) {
  if (!srs) return;
  ensure_init();  // a thread that has made no other pb200 call yet must free on the library's device
  srs_free(srs);
}
size_t pb200_srs_len(const pb200_srs_t* srs) { return srs ? srs_len(srs) : 0; }

int pb200_msm_g1_dev(const pb200_srs_t* srs, const uint64_t* d_scalars, size_t n_scalars, uint32_t batch,
                     size_t stride, uint64_t* out_affine_host, void* stream) {
  PB_TRY(ensure_init());
  if (!srs || !out_affine_host) return fail(PB200_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = stream ? (cudaStream_t)stream : thread_stream();
  return msm_run(srs, 0, d_scalars, n_scalars, batch, stride, kMsmLatency, out_affine_host, st, nullptr);
}

static int msm_host(const pb200_srs_t* srs, size_t first, const uint64_t* scalars, size_t n, uint32_t batch,
                    size_t stride, uint64_t* out) {
  PB_TRY(ensure_init());
  if (!srs || !out || (!scalars && n)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (first + n > srs_len(srs)) return fail(PB200_ERR_DEGREE_TOO_LARGE, "more scalars than commit-key points");
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint64_t* d = nullptr;
  if (n && batch) {
    PB_ALLOC(scope, d, (size_t)batch * n * 32);
    PB_CUDA(cudaMemcpy2DAsync(d, n * 32, scalars, stride * 32, n * 32, batch, cudaMemcpyHostToDevice, st));
  }
  return msm_run(srs, first, d, n, batch, n, kMsmLatency, out, st, nullptr);
}

int pb200_msm_g1(const pb200_srs_t* srs, const uint64_t* scalars, size_t n_scalars, uint32_t batch, size_t stride,
                 uint64_t* out_affine) {
  return msm_host(srs, 0, scalars, n_scalars, batch, stride, out_affine);
}
int pb200_msm_g1_range(const pb200_srs_t* srs, size_t first, const uint64_t* scalars, size_t n_scalars,
                       uint64_t* out_affine) {
  return msm_host(srs, first, scalars, n_scalars, 1, n_scalars, out_affine);
}

// ---- point-sharded MSM with an NCCL all-gather (SURVEY.md section 8e-ii, BASELINE configs[3]) ----
// NCCL is resolved at run time from the process (dlopen of libnccl.so.2: the copy the caller's
// communicator was created with when one is already loaded), so that the library itself carries no
// NCCL dependency and loads on hosts without it.
namespace {
typedef const char* (*nccl_error_string_t)(int);
struct NcclApi {
  nccl_all_gather_fn all_gather = nullptr;
  nccl_error_string_t error_string = nullptr;
};
const NcclApi* nccl_api() {
  static const NcclApi api = [] {
    NcclApi a;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (h) {
      a.all_gather = (nccl_all_gather_fn)dlsym(h, "ncclAllGather");
      a.error_string = (nccl_error_string_t)dlsym(h, "ncclGetErrorString");
    }
    return a;
  }();
  return api.all_gather ? &api : nullptr;
}
}  // namespace

static int allgather_common(const pb200_srs_t* srs_slice, const uint64_t* scalars, bool on_device, size_t n_scalars, uint32_t batch,
                            size_t stride, void* nccl_comm, int n_ranks, uint64_t* out_affine, cudaStream_t st) {
  if (!srs_slice || !out_affine || !nccl_comm || n_ranks < 1 || !batch || (!scalars && n_scalars)) return fail(PB200_ERR_INVALID_ARG, "null or empty argument");
  if (n_scalars > srs_len(srs_slice)) return fail(PB200_ERR_DEGREE_TOO_LARGE, "more scalars than commit-key points");
  const NcclApi* nccl = nccl_api();
  if (!nccl) return fail(PB200_ERR_NOT_READY, "libnccl.so.2 (ncclAllGather) is not available in this process");
  int nrc = 0;
  const int rc = msm_allgather(srs_slice, scalars, on_device, n_scalars, batch, stride, nccl->all_gather, nccl_comm, n_ranks, &nrc, out_affine, st);
  if (nrc != 0) return fail(PB200_ERR_CUDA, "ncclAllGather", nccl->error_string ? nccl->error_string(nrc) : "");
  return rc;
}

int pb200_msm_g1_allgather(const pb200_srs_t* srs_slice, const uint64_t* scalars_slice, size_t n_scalars, uint32_t batch,
                           size_t stride, void* nccl_comm, int n_ranks, uint64_t* out_affine) {
  PB_TRY(ensure_init());
  return allgather_common(srs_slice, scalars_slice, false, n_scalars, batch, stride, nccl_comm, n_ranks, out_affine, thread_stream());
}

int pb200_msm_g1_allgather_dev(const pb200_srs_t* srs_slice, const uint64_t* d_scalars_slice, size_t n_scalars, uint32_t batch,
                               size_t stride, void* nccl_comm, int n_ranks, uint64_t* out_affine_host, void* stream) {
  PB_TRY(ensure_init());
  return allgather_common(srs_slice, d_scalars_slice, true, n_scalars, batch, stride, nccl_comm, n_ranks, out_affine_host,
                          stream ? (cudaStream_t)stream : thread_stream());
}

int pb200_msm_combine_parts(const uint32_t* parts, int n_parts, int window_bits, uint32_t batch, uint64_t* out_affine,
                            size_t* words_per_entry) {
  if (window_bits < 2 || window_bits > 20 || n_parts < 0 || (parts && !out_affine)) return fail(PB200_ERR_INVALID_ARG, "bad argument");
  return msm_combine_parts(parts, n_parts, window_bits, batch, out_affine, words_per_entry);
}

int pb200_g1_compress(const uint64_t* affine_raw, uint8_t out48[48]) {
  if (!affine_raw || !out48) return fail(PB200_ERR_INVALID_ARG, "null argument");
  pbh::g1_compress_raw(affine_raw, out48);
  return 0;
}

int pb200_g1_add_affine(const uint64_t* a_raw, const uint64_t* b_raw, uint64_t* out_raw) {
  if (!a_raw || !b_raw || !out_raw) return fail(PB200_ERR_INVALID_ARG, "null argument");
  auto load = [](const uint64_t* r) {
    pbh::HXyzz p;
    memcpy(p.x.v, r, 48);
    memcpy(p.y.v, r + 6, 48);
    if (p.x.is_zero() && p.y.is_zero()) return pbh::HXyzz::identity();
    p.zz = pbh::HFp::one();
    p.zzz = pbh::HFp::one();
    return p;
  };
  pbh::HXyzz a = load(a_raw), b = load(b_raw);
  pbh::hxyzz_add(a, b);
  pbh::HFp x, y;
  pbh::hxyzz_to_affine(a, &x, &y);
  memcpy(out_raw, x.v, 48);
  memcpy(out_raw + 6, y.v, 48);
  return 0;
}

int pb200_g1_decompress(const uint8_t* compressed, size_t n_points, int check_subgroup, uint8_t* out_raw) {
  PB_TRY(ensure_init());
  if (!compressed || !out_raw) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (!n_points) return 0;
  return g1_decompress(compressed, n_points, check_subgroup, out_raw);
}

// CommitKey::to_raw_var_bytes (key.rs:215-229): u64 LE point count, then per point G1Affine::to_raw_bytes of
// dusk-bls12_381 0.14 - RAW_SIZE = 97: x, y as 6 + 6 little-endian u64 Montgomery limbs and one infinity byte.
int pb200_raw_commit_key_points(const uint8_t* bytes, size_t len, int checked, size_t* n_points) {
  if (!bytes || !n_points) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return raw_commit_key_parse(bytes, len, checked, n_points, nullptr);
}
int pb200_commit_key_from_raw_var_bytes(const uint8_t* bytes, size_t len, int checked, uint8_t* out_raw) {
  if (!bytes || !out_raw) return fail(PB200_ERR_INVALID_ARG, "null argument");
  size_t n = 0;
  PB_TRY(raw_commit_key_parse(bytes, len, checked, &n, out_raw));
  if (checked) {
    PB_TRY(ensure_init());
    PB_TRY(g1_check_raw(out_raw, n));
  }
  return 0;
}

int pb200_commit_key_to_raw_var_bytes(const uint8_t* raw_points, size_t n_points, uint8_t* out, size_t cap, size_t* len) {
  if (!len || (!raw_points && n_points)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  const size_t total = 8 + n_points * PB200_G1_RAW_SIZE;
  *len = total;
  if (!out) return 0;
  if (cap < total) return fail(PB200_ERR_INVALID_ARG, "output buffer too small");
  for (int i = 0; i < 8; i++) out[i] = (uint8_t)((uint64_t)n_points >> (8 * i));
  for (size_t i = 0; i < n_points; i++) raw_commit_key_record(raw_points + 96 * i, out + 8 + i * PB200_G1_RAW_SIZE);
  return 0;
}

int pb200_g1_compress_batch(const uint8_t* raw_points, size_t n_points, uint8_t* out_48) {
  PB_TRY(ensure_init());
  if (!n_points) return 0;
  if (!raw_points || !out_48) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return g1_compress_batch(raw_points, n_points, out_48);
}

int pb200_srs_setup_from_secret(const uint64_t* x, const uint64_t* g_scalar, size_t n_points, uint8_t* out_raw) {
  PB_TRY(ensure_init());
  if (!x || !g_scalar || !out_raw || !n_points) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return srs_setup(x, g_scalar, n_points, out_raw);
}

int pb200_public_parameters_setup(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar,
                                  uint8_t* out_raw_points, uint8_t* out_opening_key) {
  if (!out_raw_points || !out_opening_key) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(setup_args_check(max_degree, x, g_scalar, h_scalar));
  PB_TRY(ensure_init());
  const size_t n = max_degree + 7;  // max_degree + ADDED_BLINDING_DEGREE + 1 powers (srs.rs:66-79)
  PB_TRY(srs_setup(x, g_scalar, n, out_raw_points));
  uint64_t g[12];  // g = [g_scalar x^0] G, point 0 of the commit key
  memcpy(g, out_raw_points, 96);
  pbh::g1_compress_raw(g, out_opening_key);
  return opening_key_g2(x, h_scalar, out_opening_key + 48);
}

int pb200_opening_key_check(const uint8_t* opening_key) {
  if (!opening_key) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(ensure_init());
  return opening_key_check(opening_key);
}

int pb200_profile_enable(int on) {
  g_prof_acc_ns = 0; g_prof_acc_adds = 0; g_prof_acc_launches = 0; g_prof_acc_points = 0;
  g_prof_sp_ns = 0; g_prof_sp_adds = 0; g_prof_sp_launches = 0; g_prof_sp_points = 0;
  g_prof_on = on ? 1 : 0;
  return 0;
}
int pb200_profile_read(double* accumulate_ms, uint64_t* accumulate_adds, uint64_t* accumulate_launches, uint64_t* msm_points) {
  if (accumulate_ms) *accumulate_ms = (double)g_prof_acc_ns.load() * 1e-6;
  if (accumulate_adds) *accumulate_adds = g_prof_acc_adds.load();
  if (accumulate_launches) *accumulate_launches = g_prof_acc_launches.load();
  if (msm_points) *msm_points = g_prof_acc_points.load();
  return 0;
}

int pb200_profile_read_sparse(double* accumulate_ms, uint64_t* accumulate_adds, uint64_t* accumulate_launches, uint64_t* msm_points) {
  if (accumulate_ms) *accumulate_ms = (double)g_prof_sp_ns.load() * 1e-6;
  if (accumulate_adds) *accumulate_adds = g_prof_sp_adds.load();
  if (accumulate_launches) *accumulate_launches = g_prof_sp_launches.load();
  if (msm_points) *msm_points = g_prof_sp_points.load();
  return 0;
}

int pb200_g1_lagrange_key(const uint64_t* points, size_t n, uint64_t* out) {
  PB_TRY(ensure_init());
  if (!points || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (n == 0 || (n & (n - 1)) != 0) return fail(PB200_ERR_INVALID_DOMAIN, "the Lagrange key needs a power-of-two size");
  int log_n = 0;
  while (((size_t)1 << log_n) < n) log_n++;
  cudaStream_t st = thread_stream();
  uint4* buf = nullptr;  // input | output
  PB_CUDA(cudaMalloc((void**)&buf, 2 * n * 96));
  cudaError_t e = cudaMemcpyAsync(buf, points, n * 96, cudaMemcpyHostToDevice, st);
  int rc = 0;
  if (e == cudaSuccess) rc = lagrange_key_dev(buf, log_n, buf + 6 * n, st);
  if (e == cudaSuccess && rc == 0) e = cudaMemcpyAsync(out, buf + 6 * n, n * 96, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && rc == 0) e = cudaStreamSynchronize(st);
  cudaFree(buf);
  if (rc) return rc;
  PB_CUDA(e);
  return 0;
}
int pb200_imad_peak(double* mads_per_sec) {
  PB_TRY(ensure_init());
  return imad_peak(mads_per_sec);
}
int pb200_fp_product_peak(double* products_per_sec) {
  PB_TRY(ensure_init());
  if (!products_per_sec) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return fp_product_peak(products_per_sec);
}
int pb200_selftest_fr_mul(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  PB_TRY(ensure_init());
  return selftest_mul(0, a, b, out, n);
}
int pb200_selftest_fp_mul(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  PB_TRY(ensure_init());
  return selftest_mul(1, a, b, out, n);
}
int pb200_selftest_fp_ops(const uint64_t* a, const uint64_t* b, const uint64_t* c, const uint64_t* d,
                          uint64_t* out, size_t n) {
  PB_TRY(ensure_init());
  if (!a || !b || !c || !d || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return selftest_fp_ops(a, b, c, d, out, n);
}
}
