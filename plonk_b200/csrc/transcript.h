// Fiat-Shamir transcript of the prover: merlin 3.0 framing over STROBE-128 / Keccak-f[1600], plus
// the TranscriptProtocol helpers of the reference (src/transcript.rs:89-145).  Host-side product
// code (tiny, latency-bound, runs between GPU rounds); independent of oracle/.
#pragma once
#include <stdint.h>
#include <string.h>

#include "host_field.h"
#include "plonk_algebra.cuh"

namespace pbh {

inline void keccak_f1600(uint64_t s[25]) {
  static const uint64_t RC[24] = {
      0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull,
      0x000000000000808bull, 0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull,
      0x000000000000008aull, 0x0000000000000088ull, 0x0000000080008009ull, 0x000000008000000aull,
      0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull, 0x8000000000008003ull,
      0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull,
      0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};
  // rho offsets indexed [x + 5y]
  static const int RHO[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  for (int round = 0; round < 24; round++) {
    uint64_t c[5], d[5], b[25];
    for (int x = 0; x < 5; x++) c[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
    for (int x = 0; x < 5; x++) {
      const uint64_t n = c[(x + 1) % 5];
      d[x] = c[(x + 4) % 5] ^ ((n << 1) | (n >> 63));
    }
    for (int i = 0; i < 25; i++) s[i] ^= d[i % 5];
    for (int x = 0; x < 5; x++)
      for (int y = 0; y < 5; y++) {
        const int i = x + 5 * y, r = RHO[i];
        const uint64_t v = s[i];
        b[y + 5 * ((2 * x + 3 * y) % 5)] = r ? ((v << r) | (v >> (64 - r))) : v;
      }
    for (int y = 0; y < 5; y++)
      for (int x = 0; x < 5; x++) s[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
    s[0] ^= RC[round];
  }
}

class Strobe128 {
 public:
  explicit Strobe128(const char* protocol_label) {
    memset(st_, 0, sizeof st_);
    const uint8_t init[6] = {1, kRate + 2, 1, 0, 1, 96};
    memcpy(st_, init, 6);
    memcpy(st_ + 6, "STROBEv1.0.2", 12);
    permute();
    pos_ = pos_begin_ = 0;
    meta_ad((const uint8_t*)protocol_label, strlen(protocol_label), false);
  }
  void meta_ad(const uint8_t* d, size_t n, bool more) { begin_op(kM | kA, more); absorb(d, n); }
  void ad(const uint8_t* d, size_t n, bool more) { begin_op(kA, more); absorb(d, n); }
  void prf(uint8_t* out, size_t n) { begin_op(kI | kA | kC, false); squeeze(out, n); }

 private:
  enum { kRate = 166, kI = 1, kA = 2, kC = 4, kT = 8, kM = 16, kK = 32 };
  uint8_t st_[200];
  int pos_, pos_begin_;
  void permute() {
    uint64_t w[25];
    memcpy(w, st_, 200);
    keccak_f1600(w);
    memcpy(st_, w, 200);
  }
  void run_f() {
    st_[pos_] ^= (uint8_t)pos_begin_;
    st_[pos_ + 1] ^= 0x04;
    st_[kRate + 1] ^= 0x80;
    permute();
    pos_ = pos_begin_ = 0;
  }
  void absorb(const uint8_t* d, size_t n) {
    for (size_t i = 0; i < n; i++) {
      st_[pos_++] ^= d[i];
      if (pos_ == kRate) run_f();
    }
  }
  void squeeze(uint8_t* d, size_t n) {
    for (size_t i = 0; i < n; i++) {
      d[i] = st_[pos_];
      st_[pos_++] = 0;
      if (pos_ == kRate) run_f();
    }
  }
  void begin_op(int flags, bool more) {
    if (more) return;
    const uint8_t hdr[2] = {(uint8_t)pos_begin_, (uint8_t)flags};
    pos_begin_ = pos_ + 1;
    absorb(hdr, 2);
    if ((flags & (kC | kK)) && pos_ != 0) run_f();
  }
};

class Transcript {
 public:
  Transcript(const uint8_t* label, size_t n) : s_("Merlin v1.0") { append_message("dom-sep", label, n); }
  void append_message(const char* label, const uint8_t* m, size_t n) {
    const uint8_t len[4] = {(uint8_t)n, (uint8_t)(n >> 8), (uint8_t)(n >> 16), (uint8_t)(n >> 24)};
    s_.meta_ad((const uint8_t*)label, strlen(label), false);
    s_.meta_ad(len, 4, true);
    s_.ad(m, n, false);
  }
  void append_u64(const char* label, uint64_t x) {
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    append_message(label, b, 8);
  }
  // TranscriptProtocol (reference src/transcript.rs:89-108)
  void append_commitment(const char* label, const uint8_t compressed[48]) { append_message(label, compressed, 48); }
  void append_scalar(const char* label, const HFr& x) {
    HFr c = x.from_mont();
    append_message(label, (const uint8_t*)c.v, 32);
  }
  HFr challenge_scalar(const char* label) {  // 64 bytes -> BlsScalar::from_bytes_wide
    const uint8_t len[4] = {64, 0, 0, 0};
    uint8_t buf[64];
    s_.meta_ad((const uint8_t*)label, strlen(label), false);
    s_.meta_ad(len, 4, true);
    s_.prf(buf, 64);
    HFr lo, hi, r2;
    memcpy(lo.v, buf, 32);
    memcpy(hi.v, buf + 32, 32);
    memcpy(r2.v, kFrMod.r2, 32);
    const HFr r3 = r2 * r2;
    return lo * r2 + hi * r3;
  }
  void circuit_domain_sep(uint64_t n) {
    append_message("dom-sep", (const uint8_t*)"circuit_size", 12);
    append_u64("n", n);
  }

 private:
  Strobe128 s_;
};

// ---- The schedule: what goes into the transcript, in which order, under which label --------------------------
// Prover::prove_inner (prover.rs:415-761), Proof::verify (proof.rs:218-300) and Proof::verify_legacy
// (proof.rs:540-614) run the same sequence; the versions differ only in the seed.  The commitments are read from
// `comms`, the 11 compressed commitments in Proof::to_bytes order.

// VerifierKey::seed_transcript_inner (widget.rs:218-257) after Transcript::new and the constraint count.  key_comms:
// the 15 key commitments in pb::Poly order; vk_n: VerifierKey::n, which it appends last.  bind_s_sigma_4 = false
// is the legacy seed: s_sigma_1's commitment goes in under the "s_sigma_4" label (pb::kSeedOrder).
inline Transcript seed_transcript_inner(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms,
                                        uint64_t vk_n, bool bind_s_sigma_4) {
  Transcript tr(label, label_len);
  tr.circuit_domain_sep(constraints);
  for (const pb::SeedEntry& s : pb::kSeedOrder) {
    const int poly = s.poly == pb::S4 && !bind_s_sigma_4 ? pb::S1 : s.poly;
    tr.append_commitment(s.label, key_comms + 48 * poly);
  }
  tr.circuit_domain_sep(vk_n);
  return tr;
}
// Transcript::base_v3 (transcript.rs:131-145) with VerifierKey::seed_transcript: PlonkVersion::V3.
inline Transcript seed_transcript(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms, uint64_t vk_n) {
  return seed_transcript_inner(label, label_len, constraints, key_comms, vk_n, true);
}
// Transcript::base (transcript.rs:110-129) with VerifierKey::seed_transcript_legacy (widget.rs:259-265):
// PlonkVersion::V1 and V2.
inline Transcript seed_transcript_legacy(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms,
                                         uint64_t vk_n) {
  return seed_transcript_inner(label, label_len, constraints, key_comms, vk_n, false);
}
// The wire commitments -> beta, gamma.
inline void challenge_beta_gamma(Transcript& tr, const uint8_t* comms, pb::Challenges& c) {
  tr.append_commitment("a_comm", comms + 48 * pb::C_A);
  tr.append_commitment("b_comm", comms + 48 * pb::C_B);
  tr.append_commitment("c_comm", comms + 48 * pb::C_C);
  tr.append_commitment("d_comm", comms + 48 * pb::C_D);
  c.beta = tr.challenge_scalar("beta");
  tr.append_scalar("beta", c.beta);
  c.gamma = tr.challenge_scalar("gamma");
}
// The permutation commitment -> alpha and the four separation challenges.
inline void challenge_alpha(Transcript& tr, const uint8_t* comms, pb::Challenges& c) {
  tr.append_commitment("z_comm", comms + 48 * pb::C_Z);
  c.alpha = tr.challenge_scalar("alpha");
  c.range = tr.challenge_scalar("range separation challenge");
  c.logic = tr.challenge_scalar("logic separation challenge");
  c.fixed = tr.challenge_scalar("fixed base separation challenge");
  c.var = tr.challenge_scalar("variable base separation challenge");
}
// The quotient commitments -> the evaluation point z.
inline void challenge_z(Transcript& tr, const uint8_t* comms, pb::Challenges& c) {
  tr.append_commitment("t_low_comm", comms + 48 * pb::C_T_LOW);
  tr.append_commitment("t_mid_comm", comms + 48 * pb::C_T_MID);
  tr.append_commitment("t_high_comm", comms + 48 * pb::C_T_HIGH);
  tr.append_commitment("t_fourth_comm", comms + 48 * pb::C_T_FOURTH);
  c.z = tr.challenge_scalar("z_challenge");
}
// The 15 evaluations (pb::ProofEval order, Montgomery form) -> v, v_w.  They are appended in an order of their own;
// nothing is appended between the two challenges (prover.rs:680-730).
inline void challenge_v(Transcript& tr, const HFr ev[pb::N_EVAL], pb::Challenges& c) {
  static const struct {
    const char* label;
    int eval;
  } order[pb::N_EVAL] = {{"a_eval", pb::E_A},         {"b_eval", pb::E_B},         {"c_eval", pb::E_C},
                         {"d_eval", pb::E_D},         {"s_sigma_1_eval", pb::E_S1}, {"s_sigma_2_eval", pb::E_S2},
                         {"s_sigma_3_eval", pb::E_S3}, {"z_eval", pb::E_Z},          {"a_w_eval", pb::E_AW},
                         {"b_w_eval", pb::E_BW},       {"d_w_eval", pb::E_DW},       {"q_arith_eval", pb::E_QARITH},
                         {"q_c_eval", pb::E_QC},       {"q_l_eval", pb::E_QL},       {"q_r_eval", pb::E_QR}};
  for (const auto& o : order) tr.append_scalar(o.label, ev[o.eval]);
  c.v = tr.challenge_scalar("v_challenge");
  c.v_w = tr.challenge_scalar("v_w_challenge");
}
// The two opening commitments -> u (the Verifier's batching challenge; the prover stops before it).
inline void challenge_u(Transcript& tr, const uint8_t* comms, pb::Challenges& c) {
  tr.append_commitment("w_z_chall_comm", comms + 48 * pb::C_W_Z);
  tr.append_commitment("w_z_chall_w_comm", comms + 48 * pb::C_W_ZW);
  c.u = tr.challenge_scalar("u_challenge");
}

}  // namespace pbh
