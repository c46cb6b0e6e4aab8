/* plonk_b200 - C ABI of the H100-native backend for the dusk-plonk prover hot path.
 *
 * Each entry point replaces one crate-private function of the reference (paths relative to the
 * dusk-network/plonk checkout):
 *
 *   pb200_ntt / pb200_ntt_dev        EvaluationDomain::{fft, ifft, coset_fft, coset_ifft}
 *                                    src/fft/domain.rs:166-232  (best_fft :383-422)
 *   pb200_msm_g1 / pb200_msm_g1_dev  CommitKey::commit -> msm_variable_base + Commitment::from
 *                                    src/commitment_scheme/kzg10/key.rs:376-388,
 *                                    src/commitment_scheme/kzg10/commitment.rs:89-93
 *   pb200_srs_upload                 CommitKey { powers_of_g } made resident in HBM once per Prover
 *                                    src/commitment_scheme/kzg10/key.rs:36-41
 *   pb200_g1_compress                G1Affine::to_bytes as used by Commitment::to_bytes
 *                                    src/commitment_scheme/kzg10/commitment.rs:95-101
 *   pb200_g1_compress_batch          CommitKey::to_var_bytes            src/commitment_scheme/kzg10/key.rs:303-308
 *   pb200_commit_key_to_raw_var_bytes CommitKey::to_raw_var_bytes       src/commitment_scheme/kzg10/key.rs:215-229
 *   pb200_prover_* / pb200_prove     Prover::new / Prover::prove (PlonkVersion::V3)
 *                                    src/compiler/prover.rs:53-115, 415-761
 *   pb200_prover_from_bytes / _to_bytes  Prover::try_from_bytes / Prover::to_bytes
 *                                    src/compiler/prover.rs:212-350
 *   pb200_prove_with_version         Prover::prove_with_version (V2 and V3; V1 is refused as the reference does)
 *                                    src/compiler/prover.rs:364-413
 *   pb200_verifier_* / pb200_verify  Verifier / Verifier::verify (PlonkVersion::V3)
 *   pb200_verify_with_version        Verifier::verify_with_version (V1, V2 and V3)
 *                                    src/compiler/verifier.rs:32-263
 *   pb200_batch_verify               one verdict for a batch with one pairing, after OpeningKey::batch_check
 *                                    src/commitment_scheme/kzg10/key.rs:571-591, 650-707
 *   pb200_batch_verify_groups        the same over groups under several verifiers and versions (one SRS)
 *   pb200_public_parameters_setup    PublicParameters::setup      src/commitment_scheme/kzg10/srs.rs:61-100
 *   pb200_opening_key_check          OpeningKey::from_bytes       src/commitment_scheme/kzg10/key.rs:609-648
 *   pb200_circuit_compress           Circuit::compress / CompressedCircuit::from_composer
 *                                    src/composer/circuit.rs:28-45, src/composer/compress.rs:136-240
 *   pb200_compressed_circuit_info / pb200_prover_from_compressed
 *                                    Compiler::compile_with_compressed   src/compiler.rs:84-112, compress.rs:242-461
 *   pb200_pp_*                       one PublicParameters resident on the device, shared by the provers compiled from it
 *                                    src/commitment_scheme/kzg10/srs.rs:61-196
 *   pb200_circuit_unsatisfied / pb200_prover_unsatisfied / pb200_identity_family
 *                                    Debugger::unsatisfied_constraints / unsatisfied_report   src/debugger.rs:31-236
 *   (Compiler::compile, src/compiler.rs:116-461, is pb200_prover_new, pb200_prover_commitments and pb200_verifier_new
 *    in sequence; the mirrors write it once.)
 *
 * Data layout (identical to the reference's in-memory layout, SURVEY.md section 8):
 *   Fr  (BlsScalar)  4 x u64 little-endian limbs, Montgomery form R = 2^256        -> 32 bytes
 *   G1 affine        x then y, each 6 x u64 little-endian limbs, Montgomery R=2^384 -> 96 bytes;
 *                    the identity is encoded as x = y = 0.
 *
 * All functions return 0 on success or a negative pb200_status.  There is no CPU fallback: if no
 * CUDA device is usable every call fails with PB200_ERR_CUDA (the Rust shim turns that into a
 * panic, because the reference's Error enum has no device variant and the NTT functions are
 * infallible - src/error.rs:21-120, src/fft/domain.rs:394).
 * All entry points are thread safe; host-pointer variants are synchronous, *_dev variants enqueue
 * on the given CUDA stream (a cudaStream_t passed as void*, NULL = the calling thread's default
 * pb200 stream) and return without synchronising.
 */
#ifndef PLONK_B200_H
#define PLONK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  PB200_OK = 0,
  PB200_ERR_CUDA = -1,            /* CUDA runtime failure (no device, OOM, launch error) */
  PB200_ERR_INVALID_DOMAIN = -2,  /* log_n >= 32: Error::InvalidEvalDomainSize (domain.rs:132-137) */
  PB200_ERR_DEGREE_TOO_LARGE = -3,/* Error::PolynomialDegreeTooLarge (key.rs:362-370) */
  PB200_ERR_INVALID_ARG = -4,
  PB200_ERR_UNSATISFIED = -5,     /* Error::CircuitUnsatisfied (quotient_poly.rs:132-134) */
  PB200_ERR_NOT_READY = -6,
  /* -7 .. -9: circuit front end, plonk_b200_composer.h */
  PB200_ERR_POINT_MALFORMED = -10,/* dusk_bytes::Error::InvalidData / Error::PointMalformed: a G1 encoding that is
                                     not canonical, not on the curve or not in the prime-order subgroup */
  PB200_ERR_VERIFY = -11,         /* Error::ProofVerificationError: the proof does not satisfy the verifier */
  PB200_ERR_UNSUPPORTED_VERSION = -12,/* Error::UnsupportedProvingVersion: PlonkVersion::V1 proofs cannot be made */
  PB200_ERR_DEGREE_IS_ZERO = -13, /* Error::DegreeIsZero: PublicParameters::setup with max_degree = 0 (srs.rs:65-68) */
  PB200_ERR_INVALID_COMPRESSED = -14,/* Error::InvalidCompressedCircuit: a compressed circuit that does not inflate, unpack or
                                        validate within the public parameters' bounds (compress.rs:242-334) */
  PB200_ERR_SCALAR_MALFORMED = -15 /* Error::BlsScalarMalformed: a compressed circuit's scalar is not canonical (compress.rs:329-335) */
} pb200_status;

/* PlonkVersion (src/compiler.rs:22-42), for the *_with_version calls.  V3 is the current profile and the one the
 * calls without a version use.  V2 is the legacy transcript seed (Transcript::base: the commitment of s_sigma_1 goes
 * in under the "s_sigma_4" label) with V3's opening checks.  V1 is the legacy seed with the legacy opening
 * (Proof::verify_legacy, proof.rs:518-790), which does not bind the evaluations of q_arith, q_c, q_l and q_r: a V1
 * verdict is meaningful only for proofs made under the old rules, as in the reference. */
typedef enum { PB200_PLONK_V1 = 1, PB200_PLONK_V2 = 2, PB200_PLONK_V3 = 3 } pb200_plonk_version;

typedef struct pb200_srs pb200_srs_t;
typedef struct pb200_prover pb200_prover_t;
typedef struct pb200_verifier pb200_verifier_t;
typedef struct pb200_pp pb200_pp_t;

/* ---- process / device ------------------------------------------------------------------- */
/* Selects the device for this process.  Idempotent for the same device; ONE device per process: the
 * twiddle / coset tables, per-thread streams and pinned staging buffers are created on the first device
 * used, so a second call naming another device returns PB200_ERR_INVALID_ARG (multi-GPU hosts run one
 * process per GPU, as bench.py does under torchrun). */
int pb200_init(int device);
const char* pb200_last_error(void);         /* thread-local description of the last failure */
int pb200_device_sync(void);
/* Number of kernels launched by this library since process start (for bench.py's gpu_launches). */
uint64_t pb200_launch_count(void);

/* ---- NTT -------------------------------------------------------------------------------- */
/* `batch` vectors; vector b reads in + b*in_stride (in_len elements, zero padded / truncated to
 * n = 2^log_n exactly as Vec::resize does at domain.rs:174) and writes n elements at
 * out + b*out_stride.  inverse: 0 = fft, 1 = ifft (includes the 1/n scaling, domain.rs:187-196).
 * coset: 0 = plain, 1 = coset variant (distribute_powers with GENERATOR = 7 before a forward
 * transform, with 7^-1 after an inverse one; domain.rs:198-232).  Strides are in elements. */
int pb200_ntt(const uint64_t* in, size_t in_len, uint64_t* out, uint32_t log_n, int inverse,
              int coset, uint32_t batch, size_t in_stride, size_t out_stride);
int pb200_ntt_dev(const uint64_t* d_in, size_t in_len, uint64_t* d_out, uint32_t log_n,
                  int inverse, int coset, uint32_t batch, size_t in_stride, size_t out_stride,
                  void* stream);

/* ---- KZG commit key + MSM ---------------------------------------------------------------- */
/* raw_points: n_points x 96 bytes (layout above) = CommitKey::powers_of_g. */
int pb200_srs_upload(const uint8_t* raw_points, size_t n_points, pb200_srs_t** out);
/* Same with an explicit bucket-window width (bits); 0 = automatic (what pb200_srs_upload picks from
 * n_points).  The ranks of a point-sharded MSM (pb200_msm_g1_allgather*) must use ONE width for all slices:
 * take pb200_msm_window_for(largest slice) on every rank. */
int pb200_srs_upload_window(const uint8_t* raw_points, size_t n_points, int window_bits, pb200_srs_t** out);
int pb200_msm_window_for(size_t n_points);    /* the automatic choice for a key of n_points */
int pb200_srs_window(const pb200_srs_t* srs); /* the width a key was uploaded with */
void pb200_srs_free(pb200_srs_t* srs);
size_t pb200_srs_len(const pb200_srs_t* srs);

/* batch commitments sum_i scalars[b][i] * powers_of_g[i], i < n_scalars (n_scalars may be smaller
 * than the key: zip semantics of msm_variable_base).  n_scalars > pb200_srs_len() returns
 * PB200_ERR_DEGREE_TOO_LARGE.  out_affine: batch x 96 bytes, normalised affine points. */
int pb200_msm_g1(const pb200_srs_t* srs, const uint64_t* scalars, size_t n_scalars, uint32_t batch,
                 size_t stride, uint64_t* out_affine);
int pb200_msm_g1_dev(const pb200_srs_t* srs, const uint64_t* d_scalars, size_t n_scalars,
                     uint32_t batch, size_t stride, uint64_t* out_affine_host, void* stream);
/* Partial MSM over the point range [first, first + n_scalars) of the key, for sharding one large
 * MSM across GPUs by points (SURVEY.md section 8e); the caller adds the per-rank results. */
int pb200_msm_g1_range(const pb200_srs_t* srs, size_t first, const uint64_t* scalars,
                       size_t n_scalars, uint64_t* out_affine);

/* One MSM whose points are partitioned across the GPUs of a box (BASELINE.json configs[3], SURVEY.md
 * section 8e-ii): every rank calls this with its slice of the commit key (uploaded with
 * pb200_srs_upload) and the matching slice of each scalar vector (host memory, `batch` vectors of
 * stride `stride`).  The per-rank partial results - one affine point per batch entry - are exchanged
 * with a single ncclAllGather on `nccl_comm` (an ncclComm_t of `n_ranks` ranks created by the caller;
 * NCCL is looked up in the process at run time) and added locally in rank order, so every rank
 * receives the same batch x 96-byte result.  This is the only collective on the path.  (Since round 2 the
 * exchange is the device-resident one described under pb200_msm_g1_allgather_dev; this entry point only adds
 * the host -> device copy of the scalars.) */
int pb200_msm_g1_allgather(const pb200_srs_t* srs_slice, const uint64_t* scalars_slice, size_t n_scalars,
                           uint32_t batch, size_t stride, void* nccl_comm, int n_ranks, uint64_t* out_affine);
/* Same with the scalar slice already resident in HBM.  The exchange is device to device on `stream`
 * (NULL = the calling thread's pb200 stream), straight behind the reduction kernels: what travels is each
 * rank's per-digit bucket sums ((ndig + 1) x 192 bytes per batch entry plus a 16-byte header), the per-digit
 * sums are added across ranks and ONE Horner + affine normalisation finishes the result on every rank; the
 * call synchronises the stream once.  A rank whose local part fails still joins the collective (flagged in
 * its header), so its peers return PB200_ERR_CUDA instead of hanging; slices uploaded with different window
 * widths are reported as PB200_ERR_INVALID_ARG on every rank.  An empty slice (n_scalars = 0) is allowed. */
int pb200_msm_g1_allgather_dev(const pb200_srs_t* srs_slice, const uint64_t* d_scalars_slice, size_t n_scalars,
                               uint32_t batch, size_t stride, void* nccl_comm, int n_ranks,
                               uint64_t* out_affine_host, void* stream);

/* The host tail of that exchange on its own (no GPU needed): `parts` holds n_parts x batch records of
 * *words_per_entry 32-bit words - the (ndig + 1) XYZZ digit sums D_0 .. D_{ndig-1}, sum A_G a partial MSM with
 * window width `window_bits` leaves (part-major) - and out_affine receives batch x 96 bytes:
 *   R = sum_parts [ A + g * sum_j 2^shift_j D_j ],  added digit by digit, then one Horner and one shared inversion.
 * With parts = NULL only *words_per_entry is written. */
int pb200_msm_combine_parts(const uint32_t* parts, int n_parts, int window_bits, uint32_t batch,
                            uint64_t* out_affine, size_t* words_per_entry);

/* PublicParameters::setup (srs.rs:61-100).  The RNG belongs to the caller, as for pb200_prove's blinders: x, g_scalar and
 * h_scalar are the three util::random_nonzero_bls_scalar draws in the reference's order (x, then random_g1_point's scalar,
 * then random_g2_point's; util.rs:50-72), Montgomery form.  Writes max_degree + 7 raw points (max_degree +
 * ADDED_BLINDING_DEGREE + 1: out_raw_points[i] = [g_scalar * x^i] G1) and OpeningKey::to_bytes (PB200_OPENING_KEY_BYTES:
 * g = point 0 compressed, h = [h_scalar] G2 and [x] h, compressed G2 points).  The commit key is computed on the GPU by
 * fixed-base multiplication of the generator (a window table built once per process), the G2 points by one device
 * thread.  max_degree = 0 is PB200_ERR_DEGREE_IS_ZERO (Error::DegreeIsZero); a NULL pointer, a zero draw or one that is
 * not below r is PB200_ERR_INVALID_ARG; both are reported before any device is touched. */
int pb200_public_parameters_setup(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar,
                                  uint8_t* out_raw_points, uint8_t* out_opening_key);
/* OpeningKey::from_bytes (key.rs:609-648) on its own: g, h and [x]h decoded with the on-curve and subgroup checks, the
 * identity refused (OpeningKey::try_new).  PB200_OK or PB200_ERR_POINT_MALFORMED; NULL is PB200_ERR_INVALID_ARG.
 * pb200_verifier_new and pb200_verifier_from_bytes apply the same check to their opening key. */
int pb200_opening_key_check(const uint8_t* opening_key);
/* The commit-key half of pb200_public_parameters_setup with explicit secrets: out[i] = [g_scalar * x^i] G1, as
 * n_points x 96-byte raw points (the same kernel). */
int pb200_srs_setup_from_secret(const uint64_t* x, const uint64_t* g_scalar, size_t n_points,
                                uint8_t* out_raw);

/* CommitKey::from_slice / PublicParameters::from_slice (key.rs:319-326, srs.rs:163-178): decodes
 * n_points 48-byte compressed points (G1Affine::from_bytes: zcash encoding, with the on-curve and -
 * when check_subgroup != 0, as the reference always does - prime-order subgroup checks) into the
 * 96-byte raw layout pb200_srs_upload / pb200_prover_new take.  The square roots and the subgroup
 * checks run on the GPU, one thread per point.  PB200_ERR_POINT_MALFORMED names the first bad point. */
int pb200_g1_decompress(const uint8_t* compressed, size_t n_points, int check_subgroup, uint8_t* out_raw);
/* The raw ("unchecked", fast-loading) key formats of the reference - SURVEY.md section 8 row f4.
 *   CommitKey::to_raw_var_bytes (key.rs:215-229) = u64 little-endian point count, then per point
 *   G1Affine::to_raw_bytes of dusk-bls12_381 0.14: PB200_G1_RAW_SIZE = 97 bytes = x then y as 6 + 6 little-endian
 *   u64 Montgomery limbs (the first 96 bytes ARE this library's raw layout) and one byte that is 1 for the
 *   identity.  That crate is not vendored under the reference checkout and the reference holds no golden bytes
 *   for this format, so the record layout is restated from the crate's published source, not pinned by a vector.
 *   PublicParameters::to_raw_var_bytes (srs.rs:114-119) = OpeningKey::to_bytes (PB200_OPENING_KEY_BYTES = 240: a
 *   compressed G1 and two compressed G2 points, verifier material this library never reads) followed by the above.
 * checked = 0 mirrors from_slice_unchecked (key.rs:242-256, srs.rs:132-146: no point validation, at most the
 * announced count of whole records); checked = 1 mirrors CommitKey::from_raw_var_bytes (key.rs:258-298: exact
 * length, is_on_curve & is_torsion_free per point - run on the GPU; PB200_ERR_POINT_MALFORMED names the first
 * bad point).  out_raw receives n_points x 96 bytes for pb200_srs_upload / pb200_prover_new. */
#define PB200_G1_RAW_SIZE 97
#define PB200_OPENING_KEY_BYTES 240
int pb200_raw_commit_key_points(const uint8_t* bytes, size_t len, int checked, size_t* n_points);
int pb200_commit_key_from_raw_var_bytes(const uint8_t* bytes, size_t len, int checked, uint8_t* out_raw);
/* CommitKey::to_raw_var_bytes (key.rs:215-229), the writer of the format above: the u64 little-endian count, then
 * PB200_G1_RAW_SIZE bytes per point - the 96 raw bytes and a zero flag; the identity (96 zero bytes here) is written
 * as the reference's G1Affine::identity(): x = 0, y = Montgomery one, flag 1.  Host only, no device needed.
 * PublicParameters::to_raw_var_bytes (srs.rs:114-119) is this behind the 240 bytes of OpeningKey::to_bytes.
 * *len always receives 8 + n_points x 97; out = NULL writes nothing else; cap < *len is PB200_ERR_INVALID_ARG and
 * `out` is left untouched. */
int pb200_commit_key_to_raw_var_bytes(const uint8_t* raw_points, size_t n_points, uint8_t* out, size_t cap, size_t* len);
/* 48-byte compressed encoding of one affine point given in the 96-byte raw layout. */
int pb200_g1_compress(const uint64_t* affine_raw, uint8_t out48[48]);
/* CommitKey::to_var_bytes (key.rs:303-308; PublicParameters::to_var_bytes, srs.rs:149-153, is the same behind the
 * opening key): n_points x 96-byte raw points -> n_points x 48 bytes, G1Affine::to_bytes per point, byte for byte
 * what pb200_g1_compress gives.  The inverse of pb200_g1_decompress; runs on the GPU, one thread per point.
 * n_points = 0 is PB200_OK. */
int pb200_g1_compress_batch(const uint8_t* raw_points, size_t n_points, uint8_t* out_48);
/* out = a + b for two points in the 96-byte raw layout (host-side helper for multi-GPU reduction). */
int pb200_g1_add_affine(const uint64_t* a_raw, const uint64_t* b_raw, uint64_t* out_raw);

/* ---- device-resident prover (Prover::new / Prover::prove, PlonkVersion::V3) ------------------ */
/* Circuit description = what Compiler::preprocess reads from the Composer (src/compiler.rs:132-170):
 *   selectors: 11 columns x n_constraints Fr in the order q_m, q_l, q_r, q_o, q_f, q_c, q_arith,
 *              q_range, q_logic, q_fixed_group_add, q_variable_group_add (column-major);
 *   wires:     4 columns (a, b, c, d) x n_constraints witness indices;
 *   srs_raw:   PublicParameters' commit key, 96-byte raw points; it is trimmed here exactly as
 *              pp.trim(next_pow2(constraints + 6)) does (compiler.rs:121-124, srs.rs:188-196).
 * Preprocessing (15 iNTT, 15 commitments, 16 coset NTTs, sigma evaluations) runs on the GPU and
 * the prover key stays resident in HBM. */
int pb200_prover_new(const uint8_t* label, size_t label_len, size_t n_constraints,
                     const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses,
                     const uint8_t* srs_raw, size_t n_srs_points, pb200_prover_t** out);
/* Prover::try_from_bytes (src/compiler/prover.rs:265-350) for the bytes of Prover::to_bytes (:236-263): six
 * big-endian u64 (label, prover-key, commit-key, verifier-key lengths, size, constraints), the label,
 * ProverKey::to_var_bytes (src/proof_system/widget.rs:347-445: n, the byte size of one Evaluations, then for
 * each of the 15 polynomials its coefficient count, canonical 32-byte coefficients and its 8n coset
 * evaluations, then the linear and vanishing-polynomial evaluations), the commit key in the raw format above
 * and VerifierKey::to_bytes (widget.rs:84-111: n - the constraint count, compiler.rs:278-279, which try_from_bytes
 * compares with nothing and neither does this loader - and 15 compressed commitments).  The polynomials go to HBM in
 * coefficient form and the commitments are taken as stored, so none of the 15 iNTTs / 15 MSMs of preprocessing
 * runs; the 8n evaluations are recomputed by 16 coset NTTs on the device (faster than moving 17 x 8n scalars
 * over PCIe), so the serialized ones are skipped, not read.  Errors as the reference: too short ->
 * PB200_ERR_INVALID_ARG (NotEnoughBytes), inconsistent sizes / non-canonical scalars -> PB200_ERR_POINT_MALFORMED
 * (InvalidData), an invalid commit-key point -> PB200_ERR_POINT_MALFORMED (checked as try_from_bytes does).
 * A serialized Prover does not hold the circuit's wiring (the reference re-runs the circuit per proof and reads
 * the wires from that composer), so `wires` (4 x constraints witness indices) and n_witnesses come with it. */
int pb200_prover_from_bytes(const uint8_t* bytes, size_t len, const uint32_t* wires, size_t n_witnesses,
                            pb200_prover_t** out);
/* Prover::to_bytes (prover.rs:238-263) and Prover::serialized_size (:233-235): the layout pb200_prover_from_bytes
 * reads, for a prover made by pb200_prover_new or by pb200_prover_from_bytes.  Each polynomial is written with its
 * trailing zero coefficients dropped (Polynomial::from_coefficients_vec, polynomial.rs:79-93; a selector the circuit
 * never uses has length 0), the commit key is the trimmed one the prover holds (pb200_srs_len points), and
 * VerifierKey::n is the constraint count (compiler.rs:278-279).  The scalars leave HBM in chunks, converted to
 * canonical form on the device; no second copy of the key is made there.  The call reads only what the prover never
 * changes, so it may run beside proofs on the same prover; it uses the calling thread's pb200 stream.
 * *len always receives the size; out = NULL writes nothing else; cap < *len is PB200_ERR_INVALID_ARG and `out` is
 * left untouched.  The reference's Prover::try_from_bytes has not been run on these bytes (the raw point record is
 * restated, not pinned - see PB200_G1_RAW_SIZE). */
int pb200_prover_to_bytes(const pb200_prover_t* prover, uint8_t* out, size_t cap, size_t* len);
void pb200_prover_free(pb200_prover_t* prover);
/* 15 compressed commitments (verifier-key material) in the order of `selectors` then s_sigma_1..4. */
int pb200_prover_commitments(const pb200_prover_t* prover, uint8_t* out_15x48);
/* One proof.  witnesses: the Composer's witness table after running the circuit (n_witnesses Fr);
 * pi_idx / pi_vals: sorted public-input positions and values (Composer::public_input_indexes /
 * public_inputs, src/composer.rs:465-480); blinders: the 14 BlsScalar::random draws of
 * prove_inner in RNG order a0,a1,b0,b1,c0,c1,d0,d1, z0,z1,z2, b12,b13,b14 (prover.rs:154-161,
 * 503, 553-555) - the RNG belongs to the caller, as in the reference API.
 * out_proof: Proof::to_bytes, 1008 bytes (src/proof_system/proof.rs:137-162).
 * Returns PB200_ERR_UNSATISFIED for Error::CircuitUnsatisfied. */
int pb200_prove(const pb200_prover_t* prover, const uint64_t* witnesses, size_t n_witnesses,
                const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                const uint64_t* blinders, uint8_t* out_proof);
/* Same with the witness table already resident in HBM (pi_* and blinders stay host pointers);
 * n_witnesses is the length of the device table and must equal the compiled circuit's.
 * Both calls return PB200_ERR_INVALID_ARG when n_pi > 0 and pi_idx / pi_vals is NULL, when a position is
 * outside the circuit, or when pi_idx is not strictly increasing (the reference's BTreeMap cannot hold
 * duplicates).  Largest circuit: 2^28 gates (the quotient domain 8n must stay below 2^32, domain.rs:132-137). */
int pb200_prove_dev(const pb200_prover_t* prover, const uint64_t* d_witnesses, size_t n_witnesses,
                    const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                    const uint64_t* blinders, uint8_t* out_proof, void* stream);
/* Prover::prove_with_version (prover.rs:364-413): pb200_prove / pb200_prove_dev under a pb200_plonk_version.
 * PB200_PLONK_V3 is pb200_prove.  PB200_PLONK_V2 differs from it only in the transcript seed (Transcript::base);
 * the library always supports it, as the reference does with its `legacy-proving` feature on.  PB200_PLONK_V1
 * returns PB200_ERR_UNSUPPORTED_VERSION, any other value PB200_ERR_INVALID_ARG; neither touches the device. */
int pb200_prove_with_version(const pb200_prover_t* prover, int version, const uint64_t* witnesses, size_t n_witnesses,
                             const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                             const uint64_t* blinders, uint8_t* out_proof);
int pb200_prove_dev_with_version(const pb200_prover_t* prover, int version, const uint64_t* d_witnesses, size_t n_witnesses,
                                 const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                                 const uint64_t* blinders, uint8_t* out_proof, void* stream);

/* ---- which constraint a witness breaks (the reference's debugger, src/debugger.rs:31-236) ------------------------- */
/* IDENTITY_FAMILIES[k] of the reference (debugger.rs:31-49), k = 0..16: "arithmetic", the four range identities
 * ("range delta c/d", "range delta b/c", "range delta a/b", "range accumulator"), the five logic ones ("logic left
 * quad", "logic right quad", "logic output quad", "logic product", "logic relation"), the four fixed-base ones
 * ("fixed-base bit consistency", "fixed-base xy consistency", "fixed-base x accumulator", "fixed-base y accumulator")
 * and the three variable-base ones ("variable-base xy consistency", "variable-base x accumulator", "variable-base y
 * accumulator").  NULL for any other k.  No device needed. */
const char* pb200_identity_family(int k);
/* Debugger::unsatisfied_constraints (debugger.rs:95-205) on the GPU: every constraint's 17 gate identities, evaluated
 * in that order, with a_w, b_w and d_w read from row (i + 1) mod next_pow2(n_constraints) and as zero from a padding
 * row (the prover's cyclic domain).  An identity fails when it is not zero mod r; each widget identity is taken times
 * its selector, and the public input is added to the arithmetic identity outside q_arith.  This call checks a circuit
 * as pb200_prover_new takes it (selectors, wires) with its witness table and public inputs: what the composer holds at
 * prove time, which is what the reference's debugger checks.  No public parameters are needed.
 *   *n_unsatisfied always receives the number of failing constraints; rows / families receive the first min(cap, that
 *   number) of them in ascending row order, each with the index k of the first identity it fails
 *   (pb200_identity_family(k)).  With cap = 0, rows and families may be NULL.
 *   PB200_ERR_INVALID_ARG: a NULL array that is needed, public inputs that pb200_prove would refuse (positions outside
 *   the circuit or not strictly increasing), a wire index >= n_witnesses (as for pb200_prover_new).
 *   n_constraints = 0 is PB200_OK with a count of 0.
 * The call does not change when pb200_prove returns PB200_ERR_UNSATISFIED, and it checks no copy constraints: wires
 * are witness indices, so those always hold. */
int pb200_circuit_unsatisfied(size_t n_constraints, const uint64_t* selectors, const uint32_t* wires,
                              const uint64_t* witnesses, size_t n_witnesses,
                              const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                              size_t cap, uint64_t* rows, int32_t* families, size_t* n_unsatisfied);
/* The same identities against the compiled prover's own selectors, with exactly the inputs pb200_prove takes (n_witnesses
 * must be the prover's): what a proof enforces.  The selector values come from one forward NTT of the prover's key, so
 * this works for provers from pb200_prover_new, pb200_prover_from_bytes and pb200_prover_from_compressed.  Outputs and
 * argument checks as pb200_circuit_unsatisfied.  The call reads only what a prover never changes and runs on the
 * calling thread's pb200 stream, so it may run beside proofs on the same prover.  When the circuit a witness was made
 * with sets a selector the compiled one does not, pb200_circuit_unsatisfied can name a row that this call, and the
 * proof, accept; when this call reports nothing, pb200_prove makes the proof. */
int pb200_prover_unsatisfied(const pb200_prover_t* prover, const uint64_t* witnesses, size_t n_witnesses,
                             const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi,
                             size_t cap, uint64_t* rows, int32_t* families, size_t* n_unsatisfied);

/* ---- compressed circuits (Circuit::compress, Compiler::compile_with_compressed) ----------------------------------- */
/* CompressedCircuit::from_composer (src/composer/compress.rs:136-240; Circuit::compress, circuit.rs:28-45): the circuit
 * as pb200_prover_new takes it (selectors in Montgomery form, wires, the witness count) plus its public-input positions,
 * as MessagePack (layout: DESIGN.md section 2) behind raw deflate at level 9.  hades_optimization != 0 seeds the scalar
 * table with the Hades round constants and MDS entries, as Circuit::compress always does.  The inflated payload is the
 * reference's packing; the deflate bytes are zlib's, not miniz_oxide's.  Host only, no device needed.  *len always
 * receives the size; out = NULL writes nothing else; cap < *len is PB200_ERR_INVALID_ARG and `out` is left untouched.
 * A wire index >= n_witnesses or a repeated / out-of-range public-input position is PB200_ERR_INVALID_ARG.  zlib
 * (libz.so.1) is loaded at run time; without it the call is PB200_ERR_NOT_READY. */
int pb200_circuit_compress(size_t n_constraints, const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses,
                           const uint64_t* pi_idx, size_t n_pi, int hades_optimization,
                           uint8_t* out, size_t cap, size_t* len);
/* CompressedCircuit::from_bytes (compress.rs:303-450) with the bounds Compiler::compile_with_compressed derives from
 * public parameters of n_srs_points points (compiler.rs:84-112), without building anything.  In the reference's order:
 * the packed-size limit max_constraints x 857 + 30, inflation within it, unpacking with every array bounded and no
 * trailing bytes, index validation (all PB200_ERR_INVALID_COMPRESSED), then the canonical check of every serialized
 * scalar (PB200_ERR_SCALAR_MALFORMED).  Any raw-deflate stream is accepted.  Returns the gate count, the circuit's
 * witness count, n_labels (the distinct witness labels the gates use: the witnesses of the reference's rebuilt
 * composer) and the public-input count; pi_idx != NULL also receives the *n_pi positions.  Host only.  zlib as above. */
int pb200_compressed_circuit_info(const uint8_t* bytes, size_t len, size_t n_srs_points, size_t* n_constraints,
                                  uint64_t* n_witnesses, size_t* n_labels, size_t* n_pi, uint64_t* pi_idx);
/* Compiler::compile_with_compressed's Prover half: pb200_compressed_circuit_info's decoding, then Prover::new for the
 * described circuit.  Only the scalar table, the P x 11 polynomial table and one polynomial index per gate go to the
 * device, where the 11 selector columns are expanded; witness labels are renumbered densely (remap_witness,
 * compress.rs:289-301) so that host work and memory follow the gate count, never the claimed witness count.  The
 * prover keeps the circuit's own numbering: pb200_prove* take the witness table of the re-run circuit (the described
 * witness count), as for a prover from pb200_prover_new, and pb200_prover_to_bytes writes what the directly compiled
 * prover writes.  A description without gates is PB200_ERR_INVALID_ARG ("empty circuit"), as for pb200_prover_new. */
int pb200_prover_from_compressed(const uint8_t* label, size_t label_len, const uint8_t* bytes, size_t len,
                                 const uint8_t* srs_raw, size_t n_srs_points, pb200_prover_t** out);

/* ---- device-resident public parameters (one PublicParameters for many Compiler::compile calls) -------------------- */
/* A pb200_pp_t holds a PublicParameters on the device: its commit key as raw points in HBM and its opening key.  Provers
 * made from it (pb200_prover_new_pp, _from_compressed_pp, _from_bytes_pp) prove, serialize and load exactly as those
 * made from the same host points, but share the MSM tables derived from the key: the table of the trimmed key, one per
 * trimmed point count next_pow2(constraints + 6) + 7, and the Lagrange-form table, one per domain size.  Each is built
 * by the first prover that needs it (concurrent callers wait for that build; a failed build is retried by the next
 * caller) and kept until pb200_pp_free.  Provers keep the tables they use, so they may outlive the pp.  Every call may
 * run concurrently with the others on one pp except pb200_pp_free.  Too few points for a circuit is
 * PB200_ERR_DEGREE_TOO_LARGE (Error::TruncatedDegreeTooLarge). */
/* PublicParameters from raw points, as pb200_prover_new takes them (trusted, not validated), and OpeningKey::to_bytes,
 * checked as pb200_opening_key_check does (PB200_ERR_POINT_MALFORMED). */
int pb200_pp_new(const uint8_t* raw_points, size_t n_points, const uint8_t* opening_key, pb200_pp_t** out);
/* PublicParameters::setup (srs.rs:61-100) with the commit key left on the device: arguments, errors and results as
 * pb200_public_parameters_setup, and its argument errors come before any device work. */
int pb200_pp_setup(size_t max_degree, const uint64_t* x, const uint64_t* g_scalar, const uint64_t* h_scalar, pb200_pp_t** out);
/* checked = 1: PublicParameters::from_slice (srs.rs:163-178): the opening key, then 48-byte compressed points, decoded on
 * the device straight into the pp with the on-curve and subgroup checks.  checked = 0: from_slice_unchecked (srs.rs:121-146)
 * for PublicParameters::to_raw_var_bytes: the opening key, then the raw records, not validated.  The opening key is
 * checked as pb200_opening_key_check does.  Too short (at most / fewer than PB200_OPENING_KEY_BYTES) is
 * PB200_ERR_INVALID_ARG (NotEnoughBytes); a bad point, or compressed points that are not whole, PB200_ERR_POINT_MALFORMED. */
int pb200_pp_from_slice(const uint8_t* bytes, size_t len, int checked, pb200_pp_t** out);
/* The commit key's point count (PublicParameters::max_degree + 1); 0 for NULL. */
size_t pb200_pp_points(const pb200_pp_t* pp);
/* OpeningKey::to_bytes, PB200_OPENING_KEY_BYTES. */
int pb200_pp_opening_key(const pb200_pp_t* pp, uint8_t* out_240);
/* The commit key copied to the host: pb200_pp_points x 96 raw bytes. */
int pb200_pp_raw_points(const pb200_pp_t* pp, uint8_t* out_raw);
/* The derived tables the pp holds: how many trimmed-key and Lagrange-form tables, and their device bytes (any output may
 * be NULL).  A table still being built is waited for. */
int pb200_pp_tables(const pb200_pp_t* pp, size_t* n_monomial, size_t* n_lagrange, size_t* device_bytes);
/* Frees the points and the cache's references to the tables; provers made from the pp are unaffected. */
void pb200_pp_free(pb200_pp_t* pp);
/* Compiler::compile's Prover::new (src/compiler.rs:116-461) from a pp: pb200_prover_new with pp's points. */
int pb200_prover_new_pp(const pb200_pp_t* pp, const uint8_t* label, size_t label_len, size_t n_constraints,
                        const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses, pb200_prover_t** out);
/* Compiler::compile_with_compressed's Prover (src/compiler.rs:84-112) from a pp: pb200_prover_from_compressed with pp's
 * points, which also bound the decoding. */
int pb200_prover_from_compressed_pp(const pb200_pp_t* pp, const uint8_t* label, size_t label_len,
                                    const uint8_t* bytes, size_t len, pb200_prover_t** out);
/* Prover::try_from_bytes (src/compiler/prover.rs:265-350) against a pp: pb200_prover_from_bytes, except that the
 * serialized commit key must equal the pp's first points (one comparison on the device) in place of the per-point
 * validation, so the prover carries over the pp's validation.  A key that is not such a prefix is PB200_ERR_INVALID_ARG. */
int pb200_prover_from_bytes_pp(const pb200_pp_t* pp, const uint8_t* bytes, size_t len, const uint32_t* wires,
                               size_t n_witnesses, pb200_prover_t** out);

/* ---- verifier (Verifier::verify and verify_with_version; src/compiler/verifier.rs) ----------------------------- */
/* Compiler::compile's Verifier half: the label, the circuit's constraint count, the 15 verifier-key commitments in
 * pb200_prover_commitments order, OpeningKey::to_bytes (PB200_OPENING_KEY_BYTES: g compressed, then h and [x]h as
 * 96-byte compressed G2 points - zcash encoding, x.c1 then x.c0 big-endian) and the public-input positions.
 * The commitments and g are decoded with the on-curve and subgroup checks; an identity, off-curve or non-subgroup
 * opening-key point is PB200_ERR_POINT_MALFORMED (OpeningKey::try_new, key.rs:620-648).  The lines of h and [x]h
 * (G2Prepared) are computed on the device once, here. */
int pb200_verifier_new(const uint8_t* label, size_t label_len, size_t n_constraints, const uint8_t* vk_comms_15x48,
                       const uint8_t* opening_key, const uint64_t* pi_idx, size_t n_pi, pb200_verifier_t** out);
/* Verifier::try_from_bytes / Verifier::to_bytes (verifier.rs:62-202).  Layout: six big-endian u64 (label length,
 * verifier-key length = 968, opening-key length = 240, public-input count, size, constraints), the label,
 * VerifierKey::to_bytes (widget.rs:84-135: n - the constraint count, compiler.rs:278-279 - as a little-endian u64, then the commitments q_m, q_l, q_r, q_o, q_f,
 * q_c, q_arith, q_logic, q_range, q_fixed_group_add, q_variable_group_add, s_sigma_1..4 compressed, then zeros up to
 * 20 x 48 + 8 bytes), OpeningKey::to_bytes and one big-endian u64 per public-input position.  from_bytes: lengths
 * that do not fit the bytes or overflow -> PB200_ERR_INVALID_ARG (NotEnoughBytes); a malformed point ->
 * PB200_ERR_POINT_MALFORMED; a domain (the next power of two of VerifierKey::n) of 2^32 or more -> PB200_ERR_INVALID_DOMAIN.  to_bytes writes *len bytes to
 * `out` (out = NULL: only *len). */
int pb200_verifier_from_bytes(const uint8_t* bytes, size_t len, pb200_verifier_t** out);
int pb200_verifier_to_bytes(const pb200_verifier_t* verifier, uint8_t* out, size_t cap, size_t* len);
void pb200_verifier_free(pb200_verifier_t* verifier);
/* Verifier::verify for n_proofs proofs of 1008 bytes (Proof::to_bytes), each with n_pi public inputs (pi_vals:
 * n_proofs x n_pi Fr, Montgomery form).  status[i] is the proof's verdict: PB200_OK, PB200_ERR_VERIFY (the
 * pairing check fails, or z lies in the domain) or PB200_ERR_POINT_MALFORMED (Proof::from_bytes would fail: a
 * commitment that is not canonical, not on the curve or not torsion free, or a non-canonical evaluation).  A verdict
 * does not depend on the batch.  The call itself fails with PB200_ERR_INVALID_ARG when n_pi differs from the
 * verifier's public-input count (InconsistentPublicInputsLen).  pb200_verify checks PlonkVersion::V3. */
int pb200_verify(const pb200_verifier_t* verifier, const uint8_t* proofs, size_t n_proofs, const uint64_t* pi_vals,
                 size_t n_pi, int32_t* status);
/* Verifier::verify_with_version (verifier.rs:214-263): pb200_verify under a pb200_plonk_version, one version for the
 * whole batch.  Same statuses and argument checks; an unknown version is PB200_ERR_INVALID_ARG.  PB200_PLONK_V3
 * returns exactly what pb200_verify returns.  Every verifier, from pb200_verifier_new or _from_bytes, holds both
 * base transcripts, so it accepts every version.  V1 does not bind the selector evaluations (see
 * pb200_plonk_version); the device work per proof is the same for all three versions. */
int pb200_verify_with_version(const pb200_verifier_t* verifier, int version, const uint8_t* proofs, size_t n_proofs,
                              const uint64_t* pi_vals, size_t n_pi, int32_t* status);
/* Batch verification: one verdict for n_proofs proofs under one version, at the cost of one pairing.  Arguments as
 * pb200_verify_with_version.  Proof i's check e(L_i, [x]H) e(R_i, H) = 1, L_i = -(W_z + u_i W_zw), is folded into
 * e(sum w_i L_i, [x]H) e(sum w_i R_i, H) = 1 with w_i = rho^i and rho drawn, as the reference's batch_challenge
 * draws its challenge, from a merlin transcript over the whole batch: Transcript::new("dusk-plonk"), then
 * "dom-sep" = "plonk-batch-verify-v1", "version" and "batch-len" (u64) and each proof's last challenge u_i under
 * "batch-u", in batch order, and rho = challenge_scalar("batch-challenge").  A batch holding an invalid proof passes
 * with probability at most (n_proofs - 1) / r.
 * *verdict: PB200_OK when pb200_verify_with_version would give PB200_OK to every proof (up to that bound); otherwise
 * PB200_ERR_POINT_MALFORMED when some proof fails Proof::from_bytes; otherwise PB200_ERR_VERIFY.  An empty batch is
 * PB200_ERR_VERIFY, as batch_check rejects it.  The call fails with PB200_ERR_INVALID_ARG for a wrong n_pi
 * (InconsistentPublicInputsLen), an unknown version or a NULL argument, and with PB200_ERR_CUDA on a device failure. */
int pb200_batch_verify(const pb200_verifier_t* verifier, int version, const uint8_t* proofs, size_t n_proofs,
                       const uint64_t* pi_vals, size_t n_pi, int32_t* verdict);
/* Tests only: pb200_batch_verify that also returns the two folded points, sum w_i L_i then sum w_i R_i (96-byte raw
 * layout each, zeros for the identity and when the verdict is decided before the pairing). */
int pb200_selftest_batch_verify_points(const pb200_verifier_t* verifier, int version, const uint8_t* proofs, size_t n_proofs,
                                       const uint64_t* pi_vals, size_t n_pi, int32_t* verdict, uint8_t* points_2x96);
/* One verdict for several groups of proofs: group g is n_proofs[g] proofs checked under verifiers[g] and
 * versions[g], each with n_pi[g] public inputs.  proofs: every group's proofs concatenated in group order
 * (1008 bytes each); pi_vals: their public inputs concatenated in the same order (Montgomery Fr).
 * The verifiers may differ (one circuit per group, say) but must share one opening key (the same SRS), since the
 * folded check e(sum w_i L_i, [x]H) e(sum w_i R_i, H) = 1 has one pairing side; a verifier may appear in several
 * groups, for example once per version.  rho is drawn as for pb200_batch_verify, except that "version",
 * "batch-len" and the group's u_i under "batch-u" are appended once per group, in group order; w_i = rho^i over the
 * proofs in call order.  So one group gives exactly pb200_batch_verify's rho and folded points, and a call holding
 * an invalid proof passes with probability at most (N - 1) / r over its N proofs.
 * *verdict: PB200_OK when pb200_verify_with_version(verifiers[g], versions[g], ...) would give PB200_OK to every
 * proof of every group (up to that bound); otherwise PB200_ERR_POINT_MALFORMED when some proof fails
 * Proof::from_bytes; otherwise PB200_ERR_VERIFY.  No proofs at all (n_groups = 0, or every group empty) is
 * PB200_ERR_VERIFY; an empty group among others contributes nothing.  The call fails with PB200_ERR_INVALID_ARG for a
 * NULL array or verifier, an unknown version, an n_pi[g] that is not verifiers[g]'s public-input count
 * (InconsistentPublicInputsLen) or verifiers whose OpeningKey::to_bytes differ, and with PB200_ERR_CUDA on a device
 * failure. */
int pb200_batch_verify_groups(const pb200_verifier_t* const* verifiers, const int32_t* versions, const size_t* n_proofs,
                              const size_t* n_pi, size_t n_groups, const uint8_t* proofs, const uint64_t* pi_vals, int32_t* verdict);
/* Tests only: pb200_batch_verify_groups that also returns the two folded points (the layout of
 * pb200_selftest_batch_verify_points). */
int pb200_selftest_batch_verify_groups_points(const pb200_verifier_t* const* verifiers, const int32_t* versions, const size_t* n_proofs,
                                              const size_t* n_pi, size_t n_groups, const uint8_t* proofs, const uint64_t* pi_vals,
                                              int32_t* verdict, uint8_t* points_2x96);
/* Tests only: the device pairing e(P_k, Q_k) for n G1 points (96-byte raw layout) and n compressed G2 points, as
 * Fp12 values of 576 bytes (c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1; each Fp 6 x u64 Montgomery limbs). */
int pb200_selftest_pairing(const uint64_t* g1_raw, const uint8_t* g2_compressed, size_t n, uint64_t* out_fp12);

/* ---- measurement helpers ----------------------------------------------------------------- */
/* In-library CUDA-event timing of the MSM bucket-accumulation phase (k_msm_accumulate, the dominant
 * kernel of a proof, plus the two heavy-bucket kernels behind it) on its launching stream: enable resets
 * the counters; read returns the summed time, the G1 mixed additions executed (one per non-zero window
 * digit), the launch count and the MSM points processed. */
int pb200_profile_enable(int on);
/* The prover gives its dense MSMs one lane per bucket (no merge additions) as soon as two proofs are in flight on
 * it, and splits buckets over lanes for a proof that is alone (latency).  pb200_throughput_mode(1) makes single
 * proofs use the in-flight launch shape too, so that a kernel can be timed alone in the shape it has under load;
 * pb200_throughput_mode(0) restores the automatic choice.  Results never depend on it. */
int pb200_throughput_mode(int on);
int pb200_profile_read(double* accumulate_ms, uint64_t* accumulate_adds, uint64_t* accumulate_launches,
                       uint64_t* msm_points);
/* pb200_profile_read counts the DENSE MSMs (at least a quarter of the window digits non-zero: polynomial
 * coefficients); sparse ones - the wire-value commitments against the Lagrange-form key, ~1 digit per scalar,
 * mostly the over-long-bucket kernels - are accumulated separately so that they do not blur the dominant
 * kernel's rate. */
int pb200_profile_read_sparse(double* accumulate_ms, uint64_t* accumulate_adds, uint64_t* accumulate_launches,
                              uint64_t* msm_points);
/* Lagrange form of a commit key: out[j] = [L_j(x)]G = (1/n) sum_i w^(-ij) points[i] for the first
   n = 2^k points of CommitKey::powers_of_g (reference src/commitment_scheme/kzg10/key.rs:36-41), by an
   inverse NTT over group elements on the device.  Host buffers, n affine points of 96 bytes each (the
   layout of pb200_srs_upload).  With it a polynomial can be committed through its evaluations on the
   domain (sum_i p(w^i) out[i]) instead of its coefficients; the prover does not use it yet.
   PB200_ERR_INVALID_DOMAIN unless n is a power of two. */
int pb200_g1_lagrange_key(const uint64_t* points, size_t n, uint64_t* out);
/* Register-only IMAD.WIDE microbenchmark: returns achieved 32x32+64 multiply-adds per second. */
int pb200_imad_peak(double* mads_per_sec);
/* Dependent chains of carry-chained Fp (381-bit) Montgomery products, 1024 threads per SM: achieved products
 * per second - the ceiling the G1 kernels are measured against (IMAD.WIDE.U32.X, the carry-in/out form every
 * multi-limb product needs, issues at half the rate of the carry-free IMAD.WIDE that pb200_imad_peak times). */
int pb200_fp_product_peak(double* products_per_sec);
/* Elementwise Fr / Fp Montgomery products on the device (kernel self-test of the arithmetic). */
int pb200_selftest_fr_mul(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n);
int pb200_selftest_fp_mul(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n);
/* The three Fp product forms the G1 formulas use: out[0..n) = a*b, out[n..2n) = a^2,
   out[2n..3n) = a*b - c*d (6 x u64 Montgomery limbs each). */
int pb200_selftest_fp_ops(const uint64_t* a, const uint64_t* b, const uint64_t* c, const uint64_t* d,
                          uint64_t* out, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* PLONK_B200_H */
