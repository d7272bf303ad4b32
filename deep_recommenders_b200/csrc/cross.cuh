// TensorFlow's crossed_column hashing, restated for both the host compiler and sm_90a (idpipe.cu compiles it into the
// device kernel and into the host twin dr_cross_hash_host, so the two give the same ids bit for bit).
//
// tf.feature_column.crossed_column(keys, N) = tf.sparse.cross_hashed (sparse_cross_op.cc, HashCrosser):
//   * every value becomes a uint64 f: a string is FarmHash Fingerprint64 of its bytes, an int64 is used raw;
//   * dense (single-valued) inputs drop their ignore values first: the empty string, and -1 for integers.  A
//     multi-valued key is a SparseTensor there and keeps every value, '' and -1 included;
//   * for every combination of one value per key (cartesian product within the example, the LAST key varying
//     fastest, as ProductIterator enumerates it): h = hash_key; h = FingerprintCat64(h, f_key) over the keys in the
//     given order; id = h mod N on uint64.  An example in which some key has no value yields no cross.
// FingerprintCat64 is platform/fingerprint.h.  TensorFlow is not available to check this against; the CPU tests pin
// it against an independent Python restatement.
#pragma once
#include "farmhash.cuh"

#define DR_CROSS_MAX_KEYS 16

namespace dr {
namespace cross {

constexpr uint64_t kMul = 0xc6a4a7935bd1e995ull;

DR_HD uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }

DR_HD uint64_t fingerprint_cat64(uint64_t a, uint64_t b) {
  uint64_t r = a ^ kMul;
  r ^= shift_mix(b * kMul) * kMul;
  r *= kMul;
  r = shift_mix(r) * kMul;
  return shift_mix(r);
}

// One key of the cross.  values: int64 values, or (offsets != NULL) the bytes of strings delimited by offsets [n+1].
// splits: [B+1] row splits of a multi-valued key, NULL when the key has exactly one value per example.
struct Key {
  const void* values;
  const int64_t* offsets;
  const int64_t* splits;
};

struct Keys {
  Key k[DR_CROSS_MAX_KEYS];
  int n;
};

DR_HD int64_t key_begin(const Key& k, int64_t b) { return k.splits ? k.splits[b] : b; }
DR_HD int64_t key_end(const Key& k, int64_t b) { return k.splits ? k.splits[b + 1] : b + 1; }

DR_HD bool kept(const Key& k, int64_t j) {
  if (k.splits) return true;
  if (k.offsets) return k.offsets[j + 1] > k.offsets[j];
  return static_cast<const int64_t*>(k.values)[j] != -1;
}

DR_HD uint64_t value_hash(const Key& k, int64_t j) {
  if (k.offsets) {
    const int64_t o = k.offsets[j];
    return farm::fingerprint64(static_cast<const uint8_t*>(k.values) + o, (uint64_t)(k.offsets[j + 1] - o));
  }
  return (uint64_t) static_cast<const int64_t*>(k.values)[j];
}

DR_HD int64_t next_kept(const Key& k, int64_t j, int64_t end) {
  while (j < end && !kept(k, j)) ++j;
  return j;
}

// Number of crosses example b yields: the product of its kept value counts.
DR_HD int64_t count(const Keys& ks, int64_t b) {
  int64_t c = 1;
  for (int i = 0; i < ks.n && c; ++i) {
    int64_t m = 0;
    for (int64_t j = key_begin(ks.k[i], b), e = key_end(ks.k[i], b); j < e; ++j) m += kept(ks.k[i], j);
    c *= m;
  }
  return c;
}

// Writes the crosses of example b (count(ks, b) ids) to out, in TensorFlow's order.
DR_HD void fill(const Keys& ks, int64_t b, uint64_t hash_key, uint64_t num_buckets, int64_t* out) {
  int64_t pos[DR_CROSS_MAX_KEYS], end[DR_CROSS_MAX_KEYS];
  for (int i = 0; i < ks.n; ++i) {
    end[i] = key_end(ks.k[i], b);
    pos[i] = next_kept(ks.k[i], key_begin(ks.k[i], b), end[i]);
    if (pos[i] == end[i]) return;
  }
  for (int64_t o = 0;; ++o) {
    uint64_t h = hash_key;
    for (int i = 0; i < ks.n; ++i) h = fingerprint_cat64(h, value_hash(ks.k[i], pos[i]));
    out[o] = (int64_t)(h % num_buckets);
    int i = ks.n - 1;   // odometer, last key fastest
    for (; i >= 0; --i) {
      pos[i] = next_kept(ks.k[i], pos[i] + 1, end[i]);
      if (pos[i] < end[i]) break;
      pos[i] = next_kept(ks.k[i], key_begin(ks.k[i], b), end[i]);
    }
    if (i < 0) return;
  }
}

}  // namespace cross
}  // namespace dr
