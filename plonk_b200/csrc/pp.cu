// Device-resident public parameters (pb200_pp): the commit key's points in HBM, the opening key, and a cache of the
// MSM tables every prover compiled from them uses.  Also the one builder of those tables, which provers made from host
// points (pb200_prover_new, _from_bytes, _from_compressed) call for tables of their own.
//
// A prover's commit-key tables depend on the SRS and on two sizes only: the trimmed point count keep + 1 (the monomial
// table, whose length bounds a commitment's degree and is what Prover::to_bytes writes) and log n (the Lagrange form of
// the first n points).  The cache holds one entry per key, built by the first caller that needs it while later callers
// of the same key wait; an entry is published once its build has synchronised, and a failed build leaves the entry
// empty for the next caller to retry.  Entries live until pb200_pp_free; provers hold their tables by shared_ptr, so
// they may outlive the pp.
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "internal.cuh"
#include "host_field.h"

struct pb200_pp {
  struct Entry {
    std::mutex mu;  // held for the whole build: callers of the same key wait here
    std::shared_ptr<pb200_srs> table;
  };
  uint4* d_points = nullptr;  // n_points raw 96-byte points
  size_t n_points = 0;
  uint8_t opening_key[PB200_OPENING_KEY_BYTES];
  mutable std::mutex mu;                                    // guards the two maps, not the builds
  mutable std::map<size_t, std::shared_ptr<Entry>> mono;    // keyed by the point count keep + 1
  mutable std::map<int, std::shared_ptr<Entry>> lag;        // keyed by log n
};

namespace pb {

// The table over the first n_points of `points` (device or host), with the window msm_window_for(n_points).
static int monomial_table(const void* points, bool on_device, size_t n_points, std::shared_ptr<pb200_srs>* out) {
  pb200_srs* s = nullptr;
  PB_TRY(on_device ? srs_from_device((const uint4*)points, n_points, &s, 0) : srs_upload((const uint8_t*)points, n_points, &s, 0));
  out->reset(s, srs_free);
  return 0;
}

// Whether a prover over a domain of n with a trimmed key of n_points has a Lagrange-form key for its wire commitments.
static bool lagrange_wanted(size_t n, size_t n_points) {
  static const bool lagrange_env = [] {
    const char* e = getenv("PB200_LAGRANGE");
    return !e || atoi(e) != 0;
  }();
  return lagrange_env && n >= 2 && n_points >= n + 2;
}

// The Lagrange-form key of the domain of 2^log_n from the monomial points d_mono (at least n + 2 of them): n Lagrange
// points, then monomial points 0, 1, n and n + 1.
static int lagrange_table(const uint4* d_mono, int log_n, cudaStream_t st, std::shared_ptr<pb200_srs>* out) {
  const size_t n = (size_t)1 << log_n;
  uint4* comb = nullptr;  // n Lagrange points + 4 monomial ones
  PB_CUDA(cudaMalloc((void**)&comb, (n + 4) * 96));
  int rc = lagrange_key_dev(d_mono, log_n, comb, st);
  const size_t idx[4] = {0, 1, n, n + 1};
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < 4 && e == cudaSuccess; k++)
    e = cudaMemcpyAsync(comb + 6 * (n + k), d_mono + 6 * idx[k], 96, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  // Window of the Lagrange-form key.  Its scalars are witness VALUES - mostly zero or a single small digit -
  // so the bucket reduction (~2.3 additions per bucket whatever the scalars) outweighs the accumulation
  // unless the window is narrower than the monomial key's: PB200_LAG_C overrides the default.
  int lag_c = std::min(12, msm_window_for(n + 4));
  if (const char* env = getenv("PB200_LAG_C")) lag_c = atoi(env);
  if (lag_c < 2 || lag_c > 20) lag_c = 0;
  pb200_srs* s = nullptr;
  if (rc == 0 && e == cudaSuccess) rc = srs_from_device(comb, n + 4, &s, lag_c);
  cudaFree(comb);
  PB_TRY(rc);
  PB_CUDA(e);
  out->reset(s, srs_free);
  return 0;
}

int key_tables(const uint8_t* raw, size_t n_points, int log_n, cudaStream_t st, KeyTables* out) {
  PB_TRY(monomial_table(raw, false, n_points, &out->mono));
  if (lagrange_wanted((size_t)1 << log_n, n_points)) PB_TRY(lagrange_table(srs_points(out->mono.get()), log_n, st, &out->lag));
  return 0;
}

// The entry of `key` in `map`, created empty when missing.
template <class K>
static std::shared_ptr<pb200_pp::Entry> pp_entry(const pb200_pp* pp, std::map<K, std::shared_ptr<pb200_pp::Entry>>& map, K key) {
  std::lock_guard<std::mutex> lk(pp->mu);
  auto& e = map[key];
  if (!e) e = std::make_shared<pb200_pp::Entry>();
  return e;
}

// The entry's table, built by `build` unless an earlier caller has published it.
template <class F>
static int pp_cached(pb200_pp::Entry& e, std::shared_ptr<pb200_srs>* out, F&& build) {
  std::lock_guard<std::mutex> lk(e.mu);
  if (!e.table) {
    std::shared_ptr<pb200_srs> t;
    PB_TRY(build(&t));  // synchronised; nothing is published on failure
    e.table = std::move(t);
  }
  *out = e.table;
  return 0;
}

int pp_key_tables(const pb200_pp* pp, size_t n_points, int log_n, cudaStream_t st, KeyTables* out) {
  if (n_points > pp->n_points) return fail(PB200_ERR_DEGREE_TOO_LARGE, "public parameters too small for this circuit (TruncatedDegreeTooLarge)");
  PB_TRY(pp_cached(*pp_entry(pp, pp->mono, n_points), &out->mono,
                   [&](std::shared_ptr<pb200_srs>* t) { return monomial_table(pp->d_points, true, n_points, t); }));
  if (lagrange_wanted((size_t)1 << log_n, n_points))
    PB_TRY(pp_cached(*pp_entry(pp, pp->lag, log_n), &out->lag,
                     [&](std::shared_ptr<pb200_srs>* t) { return lagrange_table(pp->d_points, log_n, st, t); }));
  return 0;
}

size_t pp_points(const pb200_pp* pp) { return pp->n_points; }

// Sets *differ when a and b differ in any of their first n_words 16-byte words.
__global__ void k_points_differ(const uint4* __restrict__ a, const uint4* __restrict__ b, size_t n_words, unsigned* differ) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 x = a[i], y = b[i];
    if (x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w) {
      *differ = 1;
      return;
    }
  }
}

int pp_check_prefix(const pb200_pp* pp, const uint8_t* raw, size_t n) {
  const char* what = "the serialized prover's commit key is not a prefix of the public parameters' points";
  if (n > pp->n_points) return fail(PB200_ERR_INVALID_ARG, what);
  if (!n) return 0;
  cudaStream_t st = thread_stream();
  uint4* d = nullptr;  // n x 96 bytes, then the flag
  PB_CUDA(cudaMallocAsync((void**)&d, n * 96 + 16, st));
  unsigned* d_flag = (unsigned*)(d + 6 * n);
  unsigned differ = 0;
  cudaError_t e = cudaMemcpyAsync(d, raw, n * 96, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_flag, 0, 4, st);
  if (e == cudaSuccess) {
    const size_t words = 6 * n;
    PB_LAUNCH(k_points_differ, (unsigned)std::min<size_t>(div_up(words, 256), (size_t)num_sms() * 8), 256, 0, st, (const uint4*)d,
              (const uint4*)pp->d_points, words, d_flag);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&differ, d_flag, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFreeAsync(d, st);
  PB_CUDA(e);
  if (differ) return fail(PB200_ERR_INVALID_ARG, what);
  return 0;
}

// A pp with n points and room for them on the device; the caller fills d_points and the opening key.
static int pp_alloc(size_t n, pb200_pp** out) {
  pb200_pp* pp = new pb200_pp();
  pp->n_points = n;
  if (n) {
    const cudaError_t e = cudaMalloc((void**)&pp->d_points, n * 96);
    if (e != cudaSuccess) {
      delete pp;
      return fail(PB200_ERR_CUDA, "cudaMalloc(public parameters)", cudaGetErrorString(e));
    }
  }
  *out = pp;
  return 0;
}

static void pp_free(pb200_pp* pp) {
  cudaFree(pp->d_points);
  delete pp;  // the cache's references; provers keep the tables they hold
}

// Finishes a pp from pp_alloc: on failure it is freed and the error returned.
static int pp_finish(pb200_pp* pp, int rc, pb200_pp** out) {
  if (rc != 0) {
    pp_free(pp);
    return rc;
  }
  *out = pp;
  return 0;
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb200_pp_new(const uint8_t* raw_points, size_t n_points, const uint8_t* opening_key, pb200_pp_t** out) {
  if ((!raw_points && n_points) || !opening_key || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(ensure_init());
  PB_TRY(opening_key_check(opening_key));
  pb200_pp* pp = nullptr;
  PB_TRY(pp_alloc(n_points, &pp));
  memcpy(pp->opening_key, opening_key, PB200_OPENING_KEY_BYTES);
  int rc = 0;
  if (n_points) {
    const cudaError_t e = cudaMemcpy(pp->d_points, raw_points, n_points * 96, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) rc = fail(PB200_ERR_CUDA, "public parameters upload", cudaGetErrorString(e));
  }
  return pp_finish(pp, rc, out);
}

int pb200_pp_setup(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar, pb200_pp_t** out) {
  if (!out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(setup_args_check(max_degree, x, g_scalar, h_scalar));
  PB_TRY(ensure_init());
  const size_t n = max_degree + 7;  // max_degree + ADDED_BLINDING_DEGREE + 1 powers (srs.rs:66-79)
  pb200_pp* pp = nullptr;
  PB_TRY(pp_alloc(n, &pp));
  int rc = srs_setup_dev(x, g_scalar, n, pp->d_points);
  if (rc == 0) {
    uint64_t g[12];  // g = [g_scalar x^0] G, point 0 of the commit key
    const cudaError_t e = cudaMemcpy(g, pp->d_points, 96, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) rc = fail(PB200_ERR_CUDA, "public parameters setup", cudaGetErrorString(e));
    if (rc == 0) {
      pbh::g1_compress_raw(g, pp->opening_key);
      rc = opening_key_g2(x, h_scalar, pp->opening_key + 48);
    }
  }
  return pp_finish(pp, rc, out);
}

int pb200_pp_from_slice(const uint8_t* bytes, size_t len, int checked, pb200_pp_t** out) {
  if (!bytes || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  const size_t ok_len = PB200_OPENING_KEY_BYTES;
  if (checked ? len <= ok_len : len < ok_len) return fail(PB200_ERR_INVALID_ARG, "NotEnoughBytes: public parameters shorter than their opening key");
  if (checked && (len - ok_len) % 48) return fail(PB200_ERR_POINT_MALFORMED, "InvalidData: the commit key is not whole 48-byte points");
  PB_TRY(ensure_init());
  PB_TRY(opening_key_check(bytes));
  const uint8_t* ck = bytes + ok_len;
  const size_t ck_len = len - ok_len;
  size_t n = ck_len / 48;
  std::vector<uint8_t> raw;
  if (!checked) {
    PB_TRY(raw_commit_key_parse(ck, ck_len, 0, &n, nullptr));
    raw.resize(n * 96);
    PB_TRY(raw_commit_key_parse(ck, ck_len, 0, &n, raw.data()));
  }
  pb200_pp* pp = nullptr;
  PB_TRY(pp_alloc(n, &pp));
  memcpy(pp->opening_key, bytes, ok_len);
  if (!n) return pp_finish(pp, 0, out);
  cudaError_t e;
  unsigned bad = 0xffffffffu;
  if (checked) {  // the compressed points decoded straight into the pp, each subgroup-checked
    cudaStream_t st = thread_stream();
    uint8_t* d_in = nullptr;  // n x 48 bytes, then the index of the first bad point
    e = cudaMallocAsync((void**)&d_in, Arena::round_up(n * 48) + 16, st);
    if (e == cudaSuccess) {
      unsigned* d_bad = (unsigned*)(d_in + Arena::round_up(n * 48));
      e = cudaMemcpyAsync(d_in, ck, n * 48, cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0xff, 4, st);
      if (e == cudaSuccess) {
        g1_decompress_dev(d_in, n, pp->d_points, d_bad, st);
        e = cudaGetLastError();
      }
      if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      cudaFreeAsync(d_in, st);
    }
  } else {
    e = cudaMemcpy(pp->d_points, raw.data(), n * 96, cudaMemcpyHostToDevice);
  }
  int rc = 0;
  if (e != cudaSuccess) {
    rc = fail(PB200_ERR_CUDA, "public parameters upload", cudaGetErrorString(e));
  } else if (bad != 0xffffffffu) {
    char msg[64];
    snprintf(msg, sizeof msg, "point %u", bad);
    rc = fail(PB200_ERR_POINT_MALFORMED, "malformed G1 encoding (not canonical, not on the curve or not in the subgroup)", msg);
  }
  return pp_finish(pp, rc, out);
}

size_t pb200_pp_points(const pb200_pp_t* pp) { return pp ? pp->n_points : 0; }

int pb200_pp_opening_key(const pb200_pp_t* pp, uint8_t* out) {
  if (!pp || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  memcpy(out, pp->opening_key, PB200_OPENING_KEY_BYTES);
  return 0;
}

int pb200_pp_raw_points(const pb200_pp_t* pp, uint8_t* out_raw) {
  if (!pp || (!out_raw && pp->n_points)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (!pp->n_points) return 0;
  PB_TRY(ensure_init());
  PB_CUDA(cudaMemcpy(out_raw, pp->d_points, pp->n_points * 96, cudaMemcpyDeviceToHost));
  return 0;
}

int pb200_pp_tables(const pb200_pp_t* pp, size_t* n_monomial, size_t* n_lagrange, size_t* device_bytes) {
  if (!pp) return fail(PB200_ERR_INVALID_ARG, "null argument");
  size_t counts[2] = {0, 0}, bytes = 0;
  auto visit = [&](pb200_pp::Entry& e, int kind) {
    std::lock_guard<std::mutex> lk(e.mu);  // waits for a build in progress
    if (!e.table) return;
    const size_t c = (size_t)srs_window(e.table.get());
    counts[kind]++;
    bytes += (256 + c - 1) / c * srs_len(e.table.get()) * 96;  // W windows of the points (msm.cu's table layout)
  };
  std::vector<std::pair<std::shared_ptr<pb200_pp::Entry>, int>> entries;
  {
    std::lock_guard<std::mutex> lk(pp->mu);
    for (auto& kv : pp->mono) entries.emplace_back(kv.second, 0);
    for (auto& kv : pp->lag) entries.emplace_back(kv.second, 1);
  }
  for (auto& en : entries) visit(*en.first, en.second);
  if (n_monomial) *n_monomial = counts[0];
  if (n_lagrange) *n_lagrange = counts[1];
  if (device_bytes) *device_bytes = bytes;
  return 0;
}

void pb200_pp_free(pb200_pp_t* pp) {
  if (!pp) return;
  ensure_init();  // a thread that has made no other pb200 call yet must free on the library's device
  pp_free(pp);
}

}  // extern "C"
