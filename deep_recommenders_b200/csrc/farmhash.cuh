// FarmHash Fingerprint64 (== farmhashna::Hash64, google/farmhash, MIT licence), restated from the published
// algorithm for both the host compiler and sm_90a.  TensorFlow's categorical_column_with_hash_bucket is
// string_to_hash_bucket_fast(str(value), N) = Fingerprint64(bytes) mod N; FarmHash is a third-party dependency
// of TensorFlow, not vendored in the reference (SURVEY.md 8c).  The same source serves
//   * the device kernels of idpipe.cu (bit-exact ids are required: SURVEY 8a row E), and
//   * the host entry points dr_*_host, which the CPU tests pin against the published known answers and
//     against the independent Python restatement in deep_recommenders_b200/hashing.py.
// All arithmetic is unsigned 64-bit wrap-around; bytes are fetched one at a time (inputs are unaligned).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define DR_HD __host__ __device__ __forceinline__
#else
#define DR_HD static inline
#endif

namespace dr {
namespace farm {

constexpr uint64_t K0 = 0xC3A5C85C97CB3127ull;
constexpr uint64_t K1 = 0xB492B66FBE98F273ull;
constexpr uint64_t K2 = 0x9AE16A3B2F90404Full;

DR_HD uint64_t f64(const uint8_t* p) {
  uint64_t r = 0;
#pragma unroll
  for (int i = 7; i >= 0; --i) r = (r << 8) | (uint64_t)p[i];
  return r;
}
DR_HD uint64_t f32(const uint8_t* p) {
  return (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24);
}
DR_HD uint64_t rot(uint64_t v, int s) { return s == 0 ? v : ((v >> s) | (v << (64 - s))); }
DR_HD uint64_t smix(uint64_t v) { return v ^ (v >> 47); }

DR_HD uint64_t hl16(uint64_t u, uint64_t v, uint64_t mul) {
  uint64_t a = (u ^ v) * mul;
  a ^= (a >> 47);
  uint64_t b = (v ^ a) * mul;
  b ^= (b >> 47);
  return b * mul;
}

DR_HD uint64_t h0to16(const uint8_t* s, uint64_t n) {
  if (n >= 8) {
    const uint64_t mul = K2 + n * 2;
    const uint64_t a = f64(s) + K2;
    const uint64_t b = f64(s + n - 8);
    const uint64_t c = rot(b, 37) * mul + a;
    const uint64_t d = (rot(a, 25) + b) * mul;
    return hl16(c, d, mul);
  }
  if (n >= 4) {
    const uint64_t mul = K2 + n * 2;
    const uint64_t a = f32(s);
    return hl16(n + (a << 3), f32(s + n - 4), mul);
  }
  if (n > 0) {
    const uint8_t a = s[0], b = s[n >> 1], c = s[n - 1];
    const uint32_t y = (uint32_t)a + ((uint32_t)b << 8);
    const uint32_t z = (uint32_t)n + ((uint32_t)c << 2);
    return smix((uint64_t)y * K2 ^ (uint64_t)z * K0) * K2;
  }
  return K2;
}

DR_HD uint64_t h17to32(const uint8_t* s, uint64_t n) {
  const uint64_t mul = K2 + n * 2;
  const uint64_t a = f64(s) * K1;
  const uint64_t b = f64(s + 8);
  const uint64_t c = f64(s + n - 8) * mul;
  const uint64_t d = f64(s + n - 16) * K2;
  return hl16(rot(a + b, 43) + rot(c, 30) + d, a + rot(b + K2, 18) + c, mul);
}

DR_HD uint64_t h33to64(const uint8_t* s, uint64_t n) {
  const uint64_t mul = K2 + n * 2;
  const uint64_t a = f64(s) * K2;
  const uint64_t b = f64(s + 8);
  const uint64_t c = f64(s + n - 8) * mul;
  const uint64_t d = f64(s + n - 16) * K2;
  const uint64_t y = rot(a + b, 43) + rot(c, 30) + d;
  const uint64_t z = hl16(y, a + rot(b + K2, 18) + c, mul);
  const uint64_t e = f64(s + 16) * mul;
  const uint64_t f = f64(s + 24);
  const uint64_t g = (y + f64(s + n - 32)) * mul;
  const uint64_t h = (z + f64(s + n - 24)) * mul;
  return hl16(rot(e + f, 43) + rot(g, 30) + h, e + rot(f + a, 18) + g, mul);
}

struct Pair {
  uint64_t first, second;
};

DR_HD Pair weak32(const uint8_t* s, uint64_t a, uint64_t b) {
  const uint64_t w = f64(s), x = f64(s + 8), y = f64(s + 16), z = f64(s + 24);
  a += w;
  b = rot(b + a + z, 21);
  const uint64_t c = a;
  a += x;
  a += y;
  b += rot(a, 44);
  return Pair{a + z, b + c};
}

DR_HD uint64_t fingerprint64(const uint8_t* s, uint64_t n) {
  if (n <= 16) return h0to16(s, n);
  if (n <= 32) return h17to32(s, n);
  if (n <= 64) return h33to64(s, n);
  const uint64_t seed = 81;
  uint64_t x = seed;
  uint64_t y = seed * K1 + 113;
  uint64_t z = smix(y * K2 + 113) * K2;
  Pair v{0, 0}, w{0, 0};
  x = x * K2 + f64(s);
  const uint8_t* end = s + ((n - 1) / 64) * 64;
  const uint8_t* last64 = end + ((n - 1) & 63) - 63;
  do {
    x = rot(x + y + v.first + f64(s + 8), 37) * K1;
    y = rot(y + v.second + f64(s + 48), 42) * K1;
    x ^= w.second;
    y += v.first + f64(s + 40);
    z = rot(z + w.first, 33) * K1;
    v = weak32(s, v.second * K1, x + w.first);
    w = weak32(s + 32, z + w.second, y + f64(s + 16));
    const uint64_t t = z; z = x; x = t;
    s += 64;
  } while (s != end);
  const uint64_t mul = K1 + ((z & 0xff) << 1);
  s = last64;
  w.first += ((n - 1) & 63);
  v.first += w.first;
  w.first += v.first;
  x = rot(x + y + v.first + f64(s + 8), 37) * mul;
  y = rot(y + v.second + f64(s + 48), 42) * mul;
  x ^= w.second * 9;
  y += v.first * 9 + f64(s + 40);
  z = rot(z + w.first, 33) * mul;
  v = weak32(s, v.second * mul, x + w.first);
  w = weak32(s + 32, z + w.second, y + f64(s + 16));
  const uint64_t t = z; z = x; x = t;
  return hl16(hl16(v.first, w.first, mul) + smix(y) * K0 + z, hl16(v.second, w.second, mul) + x, mul);
}

// Decimal rendering of a signed 64-bit integer, as tf.strings.as_string(int64) produces it ("-" prefix,
// no padding): TensorFlow hashes integer features through their string form.  Returns the length (<= 20).
DR_HD int i64_to_dec(int64_t v, uint8_t* out /* >= 20 bytes */) {
  uint8_t tmp[20];
  int n = 0;
  const bool neg = v < 0;
  uint64_t u = neg ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
  do {
    tmp[n++] = (uint8_t)('0' + (u % 10));
    u /= 10;
  } while (u);
  int o = 0;
  if (neg) out[o++] = '-';
  while (n) out[o++] = tmp[--n];
  return o;
}

}  // namespace farm
}  // namespace dr
