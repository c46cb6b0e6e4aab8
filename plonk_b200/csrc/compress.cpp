// CompressedCircuit (reference src/composer/compress.rs) on the host: Circuit::compress's encoder
// (CompressedCircuit::from_composer, :136-240) and the bounded decoder of Compiler::compile_with_compressed
// (compiler.rs:84-112, compress.rs:242-461).  The payload is MessagePack as msgpacker 0.4 writes it (layout in
// DESIGN.md section 2), compressed with raw deflate.  zlib is resolved at run time (dlopen of libz.so.1), so the
// library has no link-time dependency on it.
#include "compress.h"

#include <dlfcn.h>
#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <array>
#include <mutex>
#include <string>
#include <unordered_map>

#include "../../include/plonk_b200.h"
#include "host_field.h"

namespace pb {
extern thread_local std::string g_last_error;
}

namespace pbz {

using pbh::HFr;

static int fail(int code, const std::string& what) {
  pb::g_last_error = what;
  return code;
}

// ---------------------------------------------------------------------------------------------
// zlib, resolved at run time
// ---------------------------------------------------------------------------------------------
struct Zlib {
  int (*deflate_init2)(z_streamp, int, int, int, int, int, const char*, int) = nullptr;
  int (*deflate)(z_streamp, int) = nullptr;
  int (*deflate_end)(z_streamp) = nullptr;
  uLong (*deflate_bound)(z_streamp, uLong) = nullptr;
  int (*inflate_init2)(z_streamp, int, const char*, int) = nullptr;
  int (*inflate)(z_streamp, int) = nullptr;
  int (*inflate_end)(z_streamp) = nullptr;
};

static const Zlib* zlib() {
  static const Zlib* api = [] () -> const Zlib* {
    void* h = dlopen("libz.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!h) return nullptr;
    static Zlib z;
    z.deflate_init2 = (decltype(z.deflate_init2))dlsym(h, "deflateInit2_");
    z.deflate = (decltype(z.deflate))dlsym(h, "deflate");
    z.deflate_end = (decltype(z.deflate_end))dlsym(h, "deflateEnd");
    z.deflate_bound = (decltype(z.deflate_bound))dlsym(h, "deflateBound");
    z.inflate_init2 = (decltype(z.inflate_init2))dlsym(h, "inflateInit2_");
    z.inflate = (decltype(z.inflate))dlsym(h, "inflate");
    z.inflate_end = (decltype(z.inflate_end))dlsym(h, "inflateEnd");
    if (!z.deflate_init2 || !z.deflate || !z.deflate_end || !z.deflate_bound || !z.inflate_init2 || !z.inflate || !z.inflate_end)
      return nullptr;
    return &z;
  }();
  return api;
}
static int no_zlib() { return fail(PB200_ERR_NOT_READY, "zlib (libz.so.1, raw deflate) is not available in this process"); }

// Raw deflate (no zlib header), level 9.
static int deflate_raw(const std::vector<uint8_t>& in, std::vector<uint8_t>* out) {
  const Zlib* Z = zlib();
  if (!Z) return no_zlib();
  z_stream s;
  memset(&s, 0, sizeof s);
  if (Z->deflate_init2(&s, 9, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY, ZLIB_VERSION, (int)sizeof(z_stream)) != Z_OK)
    return fail(PB200_ERR_NOT_READY, "zlib deflateInit2 failed");
  out->resize(Z->deflate_bound(&s, (uLong)in.size()) + 64);
  size_t in_at = 0, out_at = 0;
  int rc = Z_OK;
  while (rc != Z_STREAM_END) {
    if (out_at == out->size()) out->resize(2 * out->size());
    const size_t in_chunk = std::min(in.size() - in_at, (size_t)UINT32_MAX), out_chunk = std::min(out->size() - out_at, (size_t)UINT32_MAX);
    s.next_in = (Bytef*)in.data() + in_at;
    s.avail_in = (uInt)in_chunk;
    s.next_out = out->data() + out_at;
    s.avail_out = (uInt)out_chunk;
    rc = Z->deflate(&s, in_at + in_chunk == in.size() ? Z_FINISH : Z_NO_FLUSH);
    in_at += in_chunk - s.avail_in;
    out_at += out_chunk - s.avail_out;
    if (rc != Z_OK && rc != Z_STREAM_END && rc != Z_BUF_ERROR) {
      Z->deflate_end(&s);
      return fail(PB200_ERR_NOT_READY, "zlib deflate failed");
    }
  }
  Z->deflate_end(&s);
  out->resize(out_at);
  return PB200_OK;
}

// miniz_oxide::inflate::decompress_to_vec_with_limit: any raw-deflate stream whose output is at most `limit` bytes.
// The buffer grows with the output actually produced, never with a size the input claims.
static int inflate_raw(const uint8_t* in, size_t len, size_t limit, std::vector<uint8_t>* out) {
  const Zlib* Z = zlib();
  if (!Z) return no_zlib();
  z_stream s;
  memset(&s, 0, sizeof s);
  if (Z->inflate_init2(&s, -15, ZLIB_VERSION, (int)sizeof(z_stream)) != Z_OK) return fail(PB200_ERR_NOT_READY, "zlib inflateInit2 failed");
  const size_t hard = limit == SIZE_MAX ? SIZE_MAX : limit + 1;  // one byte past the limit proves it exceeded
  out->assign(std::min(hard, (size_t)1 << 16), 0);
  size_t in_at = 0, out_at = 0;
  int rc = Z_OK;
  const char* err = nullptr;
  for (;;) {
    if (out_at == out->size()) {
      if (out_at >= hard) {
        err = "InvalidCompressedCircuit: the inflated description exceeds the public parameters' size limit";
        break;
      }
      out->resize(std::min(hard, 2 * out->size()));
    }
    const size_t in_chunk = std::min(len - in_at, (size_t)UINT32_MAX), out_chunk = std::min(out->size() - out_at, (size_t)UINT32_MAX);
    s.next_in = (Bytef*)in + in_at;
    s.avail_in = (uInt)in_chunk;
    s.next_out = out->data() + out_at;
    s.avail_out = (uInt)out_chunk;
    rc = Z->inflate(&s, Z_NO_FLUSH);
    in_at += in_chunk - s.avail_in;
    out_at += out_chunk - s.avail_out;
    if (out_at > limit) {
      err = "InvalidCompressedCircuit: the inflated description exceeds the public parameters' size limit";
      break;
    }
    if (rc == Z_STREAM_END) break;
    if (rc == Z_BUF_ERROR && s.avail_out != 0) {  // no progress with room left: the input ended early
      err = "InvalidCompressedCircuit: truncated deflate stream";
      break;
    }
    if (rc != Z_OK && rc != Z_BUF_ERROR) {
      err = "InvalidCompressedCircuit: not a raw deflate stream";
      break;
    }
  }
  Z->inflate_end(&s);
  if (err) return fail(PB200_ERR_INVALID_COMPRESSED, err);
  out->resize(out_at);
  return PB200_OK;
}

// ---------------------------------------------------------------------------------------------
// SHA-512 (FIPS 180-4), for the Hades round constants
// ---------------------------------------------------------------------------------------------
static void sha512(const uint8_t* msg, size_t len, uint8_t out[64]) {
  static const uint64_t K[80] = {
      0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,
      0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,
      0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,
      0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
      0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,
      0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
      0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,
      0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
      0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,
      0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,
      0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,
      0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
      0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,
      0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,
      0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,
      0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull};
  uint64_t H[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
  auto rotr = [](uint64_t x, int n) { return (x >> n) | (x << (64 - n)); };
  std::vector<uint8_t> m(msg, msg + len);
  m.push_back(0x80);
  while (m.size() % 128 != 112) m.push_back(0);
  for (int i = 0; i < 8; i++) m.push_back(0);  // high 64 bits of the 128-bit length
  for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(((uint64_t)len * 8) >> (8 * i)));
  for (size_t blk = 0; blk < m.size(); blk += 128) {
    uint64_t w[80];
    for (int t = 0; t < 16; t++) {
      w[t] = 0;
      for (int b = 0; b < 8; b++) w[t] = (w[t] << 8) | m[blk + 8 * t + b];
    }
    for (int t = 16; t < 80; t++) {
      const uint64_t s0 = rotr(w[t - 15], 1) ^ rotr(w[t - 15], 8) ^ (w[t - 15] >> 7);
      const uint64_t s1 = rotr(w[t - 2], 19) ^ rotr(w[t - 2], 61) ^ (w[t - 2] >> 6);
      w[t] = w[t - 16] + s0 + w[t - 7] + s1;
    }
    uint64_t a = H[0], b = H[1], c = H[2], d = H[3], e = H[4], f = H[5], g = H[6], h = H[7];
    for (int t = 0; t < 80; t++) {
      const uint64_t t1 = h + (rotr(e, 14) ^ rotr(e, 18) ^ rotr(e, 41)) + ((e & f) ^ (~e & g)) + K[t] + w[t];
      const uint64_t t2 = (rotr(a, 28) ^ rotr(a, 34) ^ rotr(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
      h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    H[0] += a; H[1] += b; H[2] += c; H[3] += d; H[4] += e; H[5] += f; H[6] += g; H[7] += h;
  }
  for (int i = 0; i < 8; i++)
    for (int b = 0; b < 8; b++) out[8 * i + b] = (uint8_t)(H[i] >> (56 - 8 * b));
}

// ---------------------------------------------------------------------------------------------
// scalar_map (compress.rs:63-87): 0, 1, -1, then (hades_optimization) the Hades round constants and MDS entries not
// already present (compress/hades.rs)
// ---------------------------------------------------------------------------------------------
typedef std::array<uint64_t, 4> Key;  // a scalar's limbs (Montgomery form in the encoder, canonical in the table)
struct KeyHash {
  size_t operator()(const Key& k) const {
    uint64_t h = k[0] * 0x9e3779b97f4a7c15ull;
    h ^= (k[1] + 0x632be59bd9b4e019ull) * 0xbf58476d1ce4e5b9ull;
    h ^= (k[2] + (h >> 29)) * 0x94d049bb133111ebull;
    h ^= k[3] + (h >> 31);
    return (size_t)(h ^ (h >> 32));
  }
};
static Key key(const HFr& x) { return Key{x.v[0], x.v[1], x.v[2], x.v[3]}; }

// BlsScalar::from_bytes_wide: the 512-bit little-endian integer reduced mod r, Montgomery form
static HFr from_bytes_wide(const uint8_t b[64]) {
  HFr lo, hi, r2, r3;
  memcpy(lo.v, b, 32);
  memcpy(hi.v, b + 32, 32);
  memcpy(r2.v, pbh::kFrMod.r2, 32);
  r3 = r2 * r2;               // R^3: Montgomery products by R^2 and R^3 give lo R and hi 2^256 R
  return lo * r2 + hi * r3;   // the products reduce inputs below 2^256 (lo and hi need not be below r)
}

// The base table in Montgomery form (every entry distinct, index = position).
static const std::vector<HFr>& base_scalars(bool hades) {
  static std::once_flag once[2];
  static std::vector<HFr> table[2];
  std::call_once(once[hades], [hades] {
    std::vector<HFr>& t = table[hades];
    std::unordered_map<Key, size_t, KeyHash> seen;
    auto add = [&](const HFr& s) {
      if (seen.emplace(key(s), t.size()).second) t.push_back(s);
    };
    add(HFr::zero());
    add(HFr::one());
    add(HFr::one().neg());
    if (!hades) return;
    // 67 rounds x width 5: c_i = from_bytes_wide(SHA-512^(i+1)("poseidon-for-plonk")) + c_(i-1), c_(-1) = 1
    std::vector<uint8_t> bytes = {'p', 'o', 's', 'e', 'i', 'd', 'o', 'n', '-', 'f', 'o', 'r', '-', 'p', 'l', 'o', 'n', 'k'};
    HFr p = HFr::one();
    for (int i = 0; i < 67 * 5; i++) {
      uint8_t d[64];
      sha512(bytes.data(), bytes.size(), d);
      bytes.assign(d, d + 64);
      p = from_bytes_wide(d) + p;
      add(p);
    }
    for (int i = 0; i < 5; i++)  // the Cauchy MDS matrix: 1 / (x_i + y_j), x_i = i, y_j = j + 5
      for (int j = 0; j < 5; j++) add(HFr::from_u64(i + j + 5).inv());
  });
  return table[hades];
}

// ---------------------------------------------------------------------------------------------
// MessagePack as msgpacker 0.4 writes it: shortest unsigned integers, array headers 0x90|len / 0xdc / 0xdd, no struct
// headers, [u8; 32] as 32 bare u8
// ---------------------------------------------------------------------------------------------
struct Writer {
  std::vector<uint8_t> b;
  void be(uint64_t v, int bytes) {
    for (int i = bytes - 1; i >= 0; i--) b.push_back((uint8_t)(v >> (8 * i)));
  }
  void uint(uint64_t v) {
    if (v < 0x80) b.push_back((uint8_t)v);
    else if (v <= 0xff) { b.push_back(0xcc); be(v, 1); }
    else if (v <= 0xffff) { b.push_back(0xcd); be(v, 2); }
    else if (v <= 0xffffffffull) { b.push_back(0xce); be(v, 4); }
    else { b.push_back(0xcf); be(v, 8); }
  }
  void array(size_t len) {
    if (len <= 15) b.push_back((uint8_t)(0x90 | len));
    else if (len <= 0xffff) { b.push_back(0xdc); be(len, 2); }
    else { b.push_back(0xdd); be(len, 4); }
  }
};

struct Reader {
  const uint8_t* p;
  size_t left;
  bool take(size_t k, const uint8_t** out) {
    if (k > left) return false;
    *out = p;
    p += k;
    left -= k;
    return true;
  }
  bool be(int bytes, uint64_t* v) {
    const uint8_t* q;
    if (!take(bytes, &q)) return false;
    *v = 0;
    for (int i = 0; i < bytes; i++) *v = (*v << 8) | q[i];
    return true;
  }
  bool boolean(bool* v) {
    const uint8_t* q;
    if (!take(1, &q) || (q[0] != 0xc2 && q[0] != 0xc3)) return false;
    *v = q[0] == 0xc3;
    return true;
  }
  bool uint(uint64_t* v) {
    const uint8_t* q;
    if (!take(1, &q)) return false;
    switch (q[0]) {
      case 0xcc: return be(1, v);
      case 0xcd: return be(2, v);
      case 0xce: return be(4, v);
      case 0xcf: return be(8, v);
      default:
        if (q[0] >= 0x80) return false;
        *v = q[0];
        return true;
    }
  }
  bool u8(uint8_t* v) {
    const uint8_t* q;
    if (!take(1, &q)) return false;
    if (q[0] < 0x80) {
      *v = q[0];
      return true;
    }
    uint64_t w;
    if (q[0] != 0xcc || !be(1, &w)) return false;
    *v = (uint8_t)w;
    return true;
  }
  // PackedCircuitReader::unpack_array_len (compress.rs:496-515), then the bound of unpack_vec
  bool array(size_t max_len, size_t* len) {
    const uint8_t* q;
    if (!take(1, &q)) return false;
    uint64_t v;
    if (q[0] >= 0x90 && q[0] <= 0x9f) v = q[0] & 0x0f;
    else if (q[0] == 0xdc) { if (!be(2, &v)) return false; }
    else if (q[0] == 0xdd) { if (!be(4, &v)) return false; }
    else return false;
    if (v > max_len) return false;
    *len = (size_t)v;
    return true;
  }
};

// ---------------------------------------------------------------------------------------------
// decoding
// ---------------------------------------------------------------------------------------------
constexpr size_t kPackedFixedBytes = 30, kPackedBytesPerConstraint = 857;  // compress.rs:101-102

size_t max_constraints(size_t n_srs_points) {
  const size_t max_degree = n_srs_points ? n_srs_points - 1 : 0;
  const size_t available = max_degree > 6 ? max_degree - 6 : 0;  // ADDED_BLINDING_DEGREE
  size_t domain = 0;
  if (available) {
    domain = 1;
    while (domain <= available / 2) domain <<= 1;
  }
  return domain > 6 ? domain - 6 : 0;  // CIRCUIT_SIZE_PADDING
}

static bool canonical(const uint8_t* s) {
  for (int k = 3; k >= 0; k--) {
    uint64_t v;
    memcpy(&v, s + 8 * k, 8);
    if (v != pbh::kFrMod.p[k]) return v < pbh::kFrMod.p[k];
  }
  return false;
}

int decode(const uint8_t* bytes, size_t len, size_t n_srs_points, CompressedDescription* out) {
  const int bad = PB200_ERR_INVALID_COMPRESSED;
  // 1. the packed-size limit of the public parameters
  const size_t max_c = max_constraints(n_srs_points);
  if (max_c > (SIZE_MAX - kPackedFixedBytes) / kPackedBytesPerConstraint)
    return fail(bad, "InvalidCompressedCircuit: the packed-size limit overflows");
  const size_t limit = max_c * kPackedBytesPerConstraint + kPackedFixedBytes;
  if (max_c > SIZE_MAX / kSelectors) return fail(bad, "InvalidCompressedCircuit: the scalar-count limit overflows");
  // 2. inflate within it
  std::vector<uint8_t> packed;
  if (len && !bytes) return fail(PB200_ERR_INVALID_ARG, "null argument");
  {
    const int rc = inflate_raw(bytes, len, limit, &packed);
    if (rc) return rc;
  }
  // 3. unpack with every array bounded, nothing left over
  Reader r{packed.data(), packed.size()};
  CompressedDescription& d = *out;
  size_t n_pi = 0, n_scalars = 0, n_polys = 0, n_gates = 0;
  std::vector<uint8_t> serialized;
  std::vector<uint64_t> polys, gates;  // raw indices until they are validated
  bool ok = r.boolean(&d.hades_optimization) && r.array(max_c, &n_pi);
  if (ok) {
    d.public_inputs.resize(n_pi);
    for (size_t i = 0; ok && i < n_pi; i++) ok = r.uint(&d.public_inputs[i]);
  }
  ok = ok && r.uint(&d.witnesses) && r.array(max_c * kSelectors, &n_scalars);
  if (ok) {
    serialized.reserve(std::min(n_scalars, r.left) * 32);  // every entry takes at least 32 packed bytes
    for (size_t i = 0; ok && i < n_scalars; i++)
      for (int b = 0; ok && b < 32; b++) {
        uint8_t v = 0;
        ok = r.u8(&v);
        serialized.push_back(v);
      }
  }
  ok = ok && r.array(max_c, &n_polys);
  if (ok) {
    polys.reserve(std::min(n_polys, r.left) * kSelectors);
    for (size_t i = 0; ok && i < n_polys * kSelectors; i++) {
      uint64_t v = 0;
      ok = r.uint(&v);
      polys.push_back(v);
    }
  }
  ok = ok && r.array(max_c, &n_gates);
  if (ok) {
    gates.reserve(std::min(n_gates, r.left) * 5);
    for (size_t i = 0; ok && i < n_gates * 5; i++) {
      uint64_t v = 0;
      ok = r.uint(&v);
      gates.push_back(v);
    }
  }
  if (!ok) return fail(bad, "InvalidCompressedCircuit: malformed or oversized packed description");
  if (r.left) return fail(bad, "InvalidCompressedCircuit: trailing bytes after the packed description");
  // 4. validate_indices (compress.rs:106-134)
  const std::vector<HFr>& base = base_scalars(d.hades_optimization);
  const uint64_t scalar_count = (uint64_t)base.size() + n_scalars;
  for (size_t i = 0; i < n_pi; i++)
    if (d.public_inputs[i] >= n_gates || (i && d.public_inputs[i - 1] >= d.public_inputs[i]))
      return fail(bad, "InvalidCompressedCircuit: public-input position out of range or not increasing");
  for (uint64_t s : polys)
    if (s >= scalar_count) return fail(bad, "InvalidCompressedCircuit: scalar index out of range");
  for (size_t g = 0; g < n_gates; g++) {
    if (gates[5 * g] >= n_polys) return fail(bad, "InvalidCompressedCircuit: polynomial index out of range");
    for (int k = 1; k < 5; k++)
      if (gates[5 * g + k] >= d.witnesses) return fail(bad, "InvalidCompressedCircuit: witness index out of range");
  }
  // 5. BlsScalar::from_bytes of every serialized scalar
  for (size_t i = 0; i < n_scalars; i++)
    if (!canonical(serialized.data() + 32 * i)) return fail(PB200_ERR_SCALAR_MALFORMED, "BlsScalarMalformed: a serialized scalar is not canonical");
  if (scalar_count > UINT32_MAX) return fail(PB200_ERR_INVALID_ARG, "scalar table larger than 2^32 entries");

  d.scalars.resize(32 * scalar_count);
  for (size_t i = 0; i < base.size(); i++) memcpy(d.scalars.data() + 32 * i, base[i].from_mont().v, 32);
  if (n_scalars) memcpy(d.scalars.data() + 32 * base.size(), serialized.data(), 32 * n_scalars);
  d.polynomials.assign(polys.begin(), polys.end());
  d.gate_poly.resize(n_gates);
  d.wires.resize(4 * n_gates);
  d.labels.clear();
  // remap_witness (compress.rs:289-301): labels become dense ids in order of first appearance
  std::unordered_map<uint64_t, uint32_t> dense;
  dense.reserve(std::min(4 * n_gates, (size_t)1 << 22));
  for (size_t g = 0; g < n_gates; g++) {
    d.gate_poly[g] = (uint32_t)gates[5 * g];
    for (int k = 0; k < 4; k++) {
      const uint64_t label = gates[5 * g + 1 + k];
      auto it = dense.emplace(label, (uint32_t)d.labels.size());
      if (it.second) d.labels.push_back(label);
      d.wires[(size_t)k * n_gates + g] = it.first->second;
    }
  }
  return PB200_OK;
}

// ---------------------------------------------------------------------------------------------
// encoding: CompressedCircuit::from_composer (compress.rs:136-240)
// ---------------------------------------------------------------------------------------------
typedef std::array<uint32_t, kSelectors> Poly;
struct PolyHash {
  size_t operator()(const Poly& p) const {
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint32_t x : p) h = (h ^ x) * 0x100000001b3ull;
    return (size_t)(h ^ (h >> 29));
  }
};

static int compress(size_t n, const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses, const uint64_t* pi_idx, size_t n_pi,
                    bool hades, std::vector<uint8_t>* out) {
  for (size_t i = 0; i < 4 * n; i++)
    if (wires[i] >= n_witnesses) return fail(PB200_ERR_INVALID_ARG, "wire index out of range");
  std::vector<uint64_t> pis(pi_idx, pi_idx + n_pi);
  std::sort(pis.begin(), pis.end());
  for (size_t i = 0; i < n_pi; i++)
    if (pis[i] >= n || (i && pis[i] == pis[i - 1])) return fail(PB200_ERR_INVALID_ARG, "public-input positions out of range or repeated");

  const std::vector<HFr>& base = base_scalars(hades);
  std::vector<HFr> table(base);  // Montgomery form; keys are the limbs, a bijection of the value
  std::unordered_map<Key, uint32_t, KeyHash> scalars;
  scalars.reserve(base.size() + 1024);
  for (size_t i = 0; i < base.size(); i++) scalars.emplace(key(base[i]), (uint32_t)i);
  std::unordered_map<Poly, uint32_t, PolyHash> polys;
  std::vector<Poly> poly_list;
  std::vector<uint32_t> gate_poly(n);
  Key last[kSelectors];  // consecutive gates mostly repeat a column's value: skip the hash lookup then
  uint32_t last_idx[kSelectors];
  bool have_last[kSelectors] = {};
  for (size_t g = 0; g < n; g++) {
    Poly p;
    for (int k = 0; k < kSelectors; k++) {
      const uint64_t* s = selectors + 4 * ((size_t)k * n + g);
      const Key v{s[0], s[1], s[2], s[3]};
      if (!have_last[k] || v != last[k]) {
        auto it = scalars.emplace(v, (uint32_t)table.size());
        if (it.second) {
          HFr x;
          memcpy(x.v, s, 32);
          table.push_back(x);
        }
        last[k] = v;
        last_idx[k] = it.first->second;
        have_last[k] = true;
      }
      p[k] = last_idx[k];
    }
    auto it = polys.emplace(p, (uint32_t)poly_list.size());
    if (it.second) poly_list.push_back(p);
    gate_poly[g] = it.first->second;
  }

  Writer w;
  w.b.reserve(64 + 64 * (table.size() - base.size()) + 16 * poly_list.size() + 8 * n);
  w.b.push_back(hades ? 0xc3 : 0xc2);
  w.array(n_pi);
  for (uint64_t i : pis) w.uint(i);
  w.uint(n_witnesses);
  w.array(table.size() - base.size());  // only the scalars beyond the base table travel
  for (size_t i = base.size(); i < table.size(); i++) {
    const HFr c = table[i].from_mont();
    const uint8_t* b = (const uint8_t*)c.v;
    for (int k = 0; k < 32; k++) w.uint(b[k]);
  }
  w.array(poly_list.size());
  for (const Poly& p : poly_list)
    for (uint32_t s : p) w.uint(s);
  w.array(n);
  for (size_t g = 0; g < n; g++) {
    w.uint(gate_poly[g]);
    for (int k = 0; k < 4; k++) w.uint(wires[(size_t)k * n + g]);
  }
  return deflate_raw(w.b, out);
}

}  // namespace pbz

extern "C" {

int pb200_circuit_compress(size_t n_constraints, const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses,
                           const uint64_t* pi_idx, size_t n_pi, int hades_optimization, uint8_t* out, size_t cap, size_t* len) {
  if (!len || (n_constraints && (!selectors || !wires)) || (n_pi && !pi_idx)) return pbz::fail(PB200_ERR_INVALID_ARG, "null argument");
  std::vector<uint8_t> bytes;
  const int rc = pbz::compress(n_constraints, selectors, wires, n_witnesses, pi_idx, n_pi, hades_optimization != 0, &bytes);
  if (rc) return rc;
  *len = bytes.size();
  if (!out) return PB200_OK;
  if (cap < bytes.size()) return pbz::fail(PB200_ERR_INVALID_ARG, "output buffer too small");
  memcpy(out, bytes.data(), bytes.size());
  return PB200_OK;
}

int pb200_compressed_circuit_info(const uint8_t* bytes, size_t len, size_t n_srs_points, size_t* n_constraints,
                                  uint64_t* n_witnesses, size_t* n_labels, size_t* n_pi, uint64_t* pi_idx) {
  if (!n_constraints || !n_witnesses || !n_labels || !n_pi) return pbz::fail(PB200_ERR_INVALID_ARG, "null argument");
  pbz::CompressedDescription d;
  const int rc = pbz::decode(bytes, len, n_srs_points, &d);
  if (rc) return rc;
  *n_constraints = d.gates();
  *n_witnesses = d.witnesses;
  *n_labels = d.labels.size();
  *n_pi = d.public_inputs.size();
  if (pi_idx && !d.public_inputs.empty()) memcpy(pi_idx, d.public_inputs.data(), 8 * d.public_inputs.size());
  return PB200_OK;
}

}  // extern "C"
