// CompressedCircuit (reference src/composer/compress.rs) decoded on the host: what pb200_compressed_circuit_info reports
// and what pb200_prover_from_compressed uploads.  Host C++ only (compress.cpp); prover.cu reads the structure.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace pbz {

constexpr int kSelectors = 11;  // CompressedPolynomial: q_m, q_l, q_r, q_o, q_f, q_c, q_arith, q_range, q_logic, q_fixed_group_add, q_variable_group_add

struct CompressedDescription {
  bool hades_optimization = false;
  std::vector<uint64_t> public_inputs;  // strictly increasing gate positions
  uint64_t witnesses = 0;               // the composer's witness count: the length of the table a proof takes
  std::vector<uint8_t> scalars;         // the whole scalar table (base entries, then the serialized ones), 32 canonical bytes each
  std::vector<uint32_t> polynomials;    // P x kSelectors scalar indices
  std::vector<uint32_t> gate_poly;      // one polynomial index per gate
  std::vector<uint32_t> wires;          // [4][gates] dense witness ids (remap_witness: first appearance, gate order, a b c d)
  std::vector<uint64_t> labels;         // dense id -> the circuit's own witness index
  size_t gates() const { return gate_poly.size(); }
};

// Compiler::max_constraints (compiler.rs:101-112) for public parameters of n_srs_points points.
size_t max_constraints(size_t n_srs_points);
// CompressedCircuit::from_bytes (compress.rs:303-450) with the bounds of compile_with_compressed: PB200_OK,
// PB200_ERR_INVALID_COMPRESSED, PB200_ERR_SCALAR_MALFORMED or PB200_ERR_NOT_READY (no zlib); sets the error message.
int decode(const uint8_t* bytes, size_t len, size_t n_srs_points, CompressedDescription* out);

}  // namespace pbz
