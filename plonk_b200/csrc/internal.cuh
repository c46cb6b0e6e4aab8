// The library's internal interface: every pb:: function and global that one translation unit defines and another uses.
#pragma once
#include <memory>

#include "common.cuh"

struct pb200_srs;  // a commit key on the device (msm.cu)
struct pb200_pp;   // public parameters on the device (pp.cu)

namespace pb {

// ntt.cu
int ntt_run(const uint64_t* d_in, size_t in_len, uint64_t* d_out, uint32_t log_n, int inverse, int coset,
            uint32_t batch, size_t in_stride, size_t out_stride, cudaStream_t st, Arena* ar);
int get_twiddles(int logm, bool inverse, cudaStream_t st, const uint4** out);
int fill_powers(uint4* out, size_t n, const Fr& base, const Fr& scale, cudaStream_t st);
Fr ntt_group_gen(int log_n, bool inverse);
Fr ntt_size_inv(int log_n);
Fr ntt_coset_gen(bool inverse);

// msm.cu.  The launch shape of an MSM is its caller's choice.  split_buckets: several lanes per bucket while the buckets
// alone cannot fill the GPU (latency for an MSM that is alone; the merge additions are lost work once other proofs keep
// the GPU busy).  wide_heavy_chunks: over-long buckets are summed 32 entries per lane instead of 8 (fewer tree additions).
struct MsmShape {
  bool split_buckets, wide_heavy_chunks;
};
constexpr MsmShape kMsmLatency = {true, false};  // an MSM alone on the GPU
int msm_run(const pb200_srs* srs, size_t first, const uint64_t* d_scalars, size_t n, uint32_t batch, size_t stride,
            MsmShape shape, uint64_t* out_affine_host, cudaStream_t st, Arena* ar);
size_t msm_workspace_bytes(const pb200_srs* srs, size_t n, uint32_t batch);
typedef int (*nccl_all_gather_fn)(const void*, void*, size_t, int, void*, cudaStream_t);  // ncclAllGather
int msm_allgather(const pb200_srs* srs, const uint64_t* scalars, bool scalars_on_device, size_t n, uint32_t batch, size_t stride,
                  nccl_all_gather_fn all_gather, void* comm, int n_ranks, int* nccl_rc, uint64_t* out_affine_host, cudaStream_t st);
int msm_combine_parts(const uint32_t* parts, int n_parts, int window_bits, uint32_t batch, uint64_t* out_affine_host, size_t* words_per_entry);
int msm_window_for(size_t n_points);
int srs_upload(const uint8_t* raw, size_t n_points, pb200_srs** out, int window_bits);  // window_bits 0: msm_window_for
int srs_from_device(const uint4* d_points, size_t n_points, pb200_srs** out, int window_bits);
const uint4* srs_points(const pb200_srs* s);
size_t srs_len(const pb200_srs* s);
int srs_window(const pb200_srs* s);
void srs_free(pb200_srs* s);
int srs_setup(const uint64_t* x_mont, const uint64_t* g_scalar_mont, size_t n, uint8_t* out_raw);
int srs_setup_dev(const uint64_t* x_mont, const uint64_t* g_scalar_mont, size_t n, uint4* d_out);  // n x 96 bytes, synchronised
int g1_decompress(const uint8_t* in, size_t n, int check_subgroup, uint8_t* out_raw);
void g1_decompress_dev(const uint8_t* d_in, size_t n, uint4* d_out, unsigned* d_bad, cudaStream_t st);
int g1_check_raw(const uint8_t* raw, size_t n);
int g1_compress_batch(const uint8_t* raw, size_t n, uint8_t* out_48);
int selftest_mul(int which, const uint64_t* a, const uint64_t* b, uint64_t* o, size_t n);
int selftest_fp_ops(const uint64_t* a, const uint64_t* b, const uint64_t* c, const uint64_t* d, uint64_t* o, size_t n);
int imad_peak(double* out);
int fp_product_peak(double* out);
extern std::atomic<int> g_prof_on;  // bucket-accumulation timing (pb200_profile_*): dense and sparse MSMs
extern std::atomic<uint64_t> g_prof_acc_ns, g_prof_acc_adds, g_prof_acc_launches, g_prof_acc_points;
extern std::atomic<uint64_t> g_prof_sp_ns, g_prof_sp_adds, g_prof_sp_launches, g_prof_sp_points;

// ecntt.cu
int lagrange_key_dev(const uint4* d_in, int log_n, uint4* d_out, cudaStream_t st);

// verify.cu: OpeningKey::from_bytes's checks alone, and the G2 half of PublicParameters::setup (h, then [x]h, compressed)
int opening_key_check(const uint8_t* opening_key);
int opening_key_g2(const uint64_t* x_mont, const uint64_t* h_scalar_mont, uint8_t* out_2x96);

// debugger.cu: the reference debugger's row check over columns already on the device (sel [11][n] selector values,
// wv [4][n] wire values zero-padded past the constraints, pi [n] or null); writes the total to *n_unsatisfied and the
// first min(cap, total) failing rows and their identity indices to the host arrays rows / families.  Synchronises st.
int unsatisfied_run(const uint4* sel, const uint4* wv, const uint4* pi, size_t n, size_t constraints, size_t cap, uint64_t* rows,
                    int32_t* families, size_t* n_unsatisfied, cudaStream_t st);

// pp.cu: the MSM tables of one prover's commit key - the monomial table over its trimmed n_points and, for most
// domains, the Lagrange-form table of the domain of 2^log_n - built from host points for this prover alone (key_tables)
// or taken from the pp's cache (pp_key_tables, PB200_ERR_DEGREE_TOO_LARGE when n_points exceeds the pp's).
struct KeyTables {
  std::shared_ptr<pb200_srs> mono, lag;  // lag is null when the prover commits its wires with the monomial table
};
int key_tables(const uint8_t* raw, size_t n_points, int log_n, cudaStream_t st, KeyTables* out);
int pp_key_tables(const pb200_pp* pp, size_t n_points, int log_n, cudaStream_t st, KeyTables* out);
size_t pp_points(const pb200_pp* pp);
// PB200_ERR_INVALID_ARG unless the n host raw points are the pp's first n
int pp_check_prefix(const pb200_pp* pp, const uint8_t* raw, size_t n);

// capi.cu
int setup_args_check(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar);
int raw_commit_key_parse(const uint8_t* bytes, size_t len, int checked, size_t* n_points, uint8_t* out_raw);
void raw_commit_key_record(const uint8_t* raw96, uint8_t* rec97);

}  // namespace pb
