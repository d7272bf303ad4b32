// SURVEY.md 8(f) #2 -- the id pipeline in front of the gather: raw feature value -> int64 row id.
//   categorical_column_with_hash_bucket      id = FarmHash Fingerprint64(str(value)) mod N
//   categorical_column_with_vocabulary_list  id = position in the list, out-of-vocabulary -> default (-1)
//   crossed_column                           id = FingerprintCat64 chain over the keys' values mod N (cross.cuh)
// (reference call sites: examples/train_deepfm_on_movielens_keras.py:12-24; the arithmetic is TensorFlow's.)
// Integer / byte work: results must be bit-exact, so the device kernels and the host twins compile the same
// farmhash.cuh.  One thread per value: the work is a few hundred integer ops on <= 20 bytes per id, far below
// the HBM time of the gather that follows.
#include "common.cuh"
#include "farmhash.cuh"
#include "cross.cuh"

namespace dr {

__global__ void __launch_bounds__(256) hash_bucket_i64_kernel(const int64_t* __restrict__ values, int64_t n,
                                                               uint64_t num_buckets, int64_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint8_t buf[20];
    const int len = farm::i64_to_dec(__ldg(values + i), buf);
    out[i] = (int64_t)(farm::fingerprint64(buf, (uint64_t)len) % num_buckets);
  }
}

__global__ void __launch_bounds__(256) hash_bucket_bytes_kernel(const uint8_t* __restrict__ bytes,
                                                                 const int64_t* __restrict__ offsets, int64_t n,
                                                                 uint64_t num_buckets, int64_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t b = __ldg(offsets + i), e = __ldg(offsets + i + 1);
    out[i] = (int64_t)(farm::fingerprint64(bytes + b, (uint64_t)(e - b)) % num_buckets);
  }
}

// Vocabulary lookup on integer keys: binary search in the key-sorted copy of the list; vocab_index[j] is the
// position of keys_sorted[j] in the user's list.
__global__ void __launch_bounds__(256) vocab_lookup_i64_kernel(const int64_t* __restrict__ values, int64_t n,
                                                                const int64_t* __restrict__ keys_sorted,
                                                                const int64_t* __restrict__ vocab_index,
                                                                int64_t vocab_size, int64_t default_id,
                                                                int64_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t v = __ldg(values + i);
    int64_t lo = 0, hi = vocab_size;   // first key >= v
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(keys_sorted + mid) < v) lo = mid + 1; else hi = mid;
    }
    out[i] = (lo < vocab_size && __ldg(keys_sorted + lo) == v) ? __ldg(vocab_index + lo) : default_id;
  }
}

// crossed_column (cross.cuh), one thread per example.  out_splits == NULL: every key is single-valued and out_ids[b]
// is the example's one cross, or -1 when a key's value is an ignore value.  out_ids == NULL: out_splits[b + 1] = the
// number of crosses of example b (the caller turns the counts into row splits).  Otherwise the crosses of b go to
// out_ids[out_splits[b] ..].
__global__ void __launch_bounds__(256) cross_hash_kernel(const cross::Keys ks, int64_t B, uint64_t hash_key,
                                                          uint64_t num_buckets, int64_t* __restrict__ out_splits,
                                                          int64_t* __restrict__ out_ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += stride) {
    if (!out_splits) {
      if (cross::count(ks, b) == 1) cross::fill(ks, b, hash_key, num_buckets, out_ids + b);
      else out_ids[b] = -1;
    } else if (!out_ids) {
      out_splits[b + 1] = cross::count(ks, b);
      if (b == 0) out_splits[0] = 0;
    } else {
      cross::fill(ks, b, hash_key, num_buckets, out_ids + out_splits[b]);
    }
  }
}

static inline unsigned grid_for(int64_t n) {
  int64_t ctas = (n + 255) / 256;
  if (ctas > num_sms() * 8) ctas = num_sms() * 8;
  return (unsigned)(ctas < 1 ? 1 : ctas);
}

}  // namespace dr

using namespace dr;

extern "C" uint64_t dr_fingerprint64_host(const uint8_t* s, int64_t len) {
  return farm::fingerprint64(s, (uint64_t)(len < 0 ? 0 : len));
}

extern "C" int dr_hash_bucket_bytes_host(const uint8_t* bytes, const int64_t* offsets, int64_t n,
                                         int64_t num_buckets, int64_t* out_ids) {
  DR_REQUIRE(offsets && out_ids && (bytes || n == 0), DR_EINVAL, "dr_hash_bucket_bytes_host: null pointer");
  DR_REQUIRE(n >= 0 && num_buckets >= 1, DR_EINVAL, "dr_hash_bucket_bytes_host: n=%lld num_buckets=%lld",
             (long long)n, (long long)num_buckets);
  for (int64_t i = 0; i < n; ++i) {
    DR_REQUIRE(offsets[i + 1] >= offsets[i], DR_EINVAL, "dr_hash_bucket_bytes_host: offsets not monotone at %lld",
               (long long)i);
    out_ids[i] = (int64_t)(farm::fingerprint64(bytes + offsets[i], (uint64_t)(offsets[i + 1] - offsets[i])) %
                           (uint64_t)num_buckets);
  }
  return DR_OK;
}

extern "C" int dr_hash_bucket_i64_host(const int64_t* values, int64_t n, int64_t num_buckets, int64_t* out_ids) {
  DR_REQUIRE((values && out_ids) || n == 0, DR_EINVAL, "dr_hash_bucket_i64_host: null pointer");
  DR_REQUIRE(n >= 0 && num_buckets >= 1, DR_EINVAL, "dr_hash_bucket_i64_host: n=%lld num_buckets=%lld",
             (long long)n, (long long)num_buckets);
  for (int64_t i = 0; i < n; ++i) {
    uint8_t buf[20];
    const int len = farm::i64_to_dec(values[i], buf);
    out_ids[i] = (int64_t)(farm::fingerprint64(buf, (uint64_t)len) % (uint64_t)num_buckets);
  }
  return DR_OK;
}

extern "C" int dr_hash_bucket_i64(const int64_t* values, int64_t n, int64_t num_buckets, int64_t* out_ids,
                                  void* stream) {
  DR_REQUIRE(n >= 0 && num_buckets >= 1, DR_EINVAL, "dr_hash_bucket_i64: n=%lld num_buckets=%lld", (long long)n,
             (long long)num_buckets);
  if (n == 0) return DR_OK;
  DR_REQUIRE(values && out_ids, DR_EINVAL, "dr_hash_bucket_i64: null pointer");
  hash_bucket_i64_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(values, n, (uint64_t)num_buckets, out_ids);
  DR_CUDA_LAUNCH_CHECK("hash_bucket_i64");
  return DR_OK;
}

extern "C" int dr_hash_bucket_bytes(const uint8_t* bytes, const int64_t* offsets, int64_t n, int64_t num_buckets,
                                    int64_t* out_ids, void* stream) {
  DR_REQUIRE(n >= 0 && num_buckets >= 1, DR_EINVAL, "dr_hash_bucket_bytes: n=%lld num_buckets=%lld", (long long)n,
             (long long)num_buckets);
  if (n == 0) return DR_OK;
  DR_REQUIRE(bytes && offsets && out_ids, DR_EINVAL, "dr_hash_bucket_bytes: null pointer");
  hash_bucket_bytes_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(bytes, offsets, n, (uint64_t)num_buckets,
                                                                           out_ids);
  DR_CUDA_LAUNCH_CHECK("hash_bucket_bytes");
  return DR_OK;
}

extern "C" int dr_vocab_lookup_i64(const int64_t* values, int64_t n, const int64_t* keys_sorted,
                                   const int64_t* vocab_index, int64_t vocab_size, int64_t default_id,
                                   int64_t* out_ids, void* stream) {
  DR_REQUIRE(n >= 0 && vocab_size >= 1, DR_EINVAL, "dr_vocab_lookup_i64: n=%lld vocab_size=%lld", (long long)n,
             (long long)vocab_size);
  if (n == 0) return DR_OK;
  DR_REQUIRE(values && keys_sorted && vocab_index && out_ids, DR_EINVAL, "dr_vocab_lookup_i64: null pointer");
  vocab_lookup_i64_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(values, n, keys_sorted, vocab_index,
                                                                          vocab_size, default_id, out_ids);
  DR_CUDA_LAUNCH_CHECK("vocab_lookup_i64");
  return DR_OK;
}

namespace dr {
// Validates the arguments shared by dr_cross_hash and its host twin and packs the keys.
static int cross_keys(int K, const void* const* values, const int64_t* const* value_offsets,
                      const int64_t* const* row_splits, int64_t B, int64_t num_buckets, const int64_t* out_splits,
                      const int64_t* out_ids, const char* who, cross::Keys* ks) {
  DR_REQUIRE(K >= 2 && K <= DR_CROSS_MAX_KEYS, DR_EINVAL, "%s: K=%d keys (need 2..%d)", who, K, DR_CROSS_MAX_KEYS);
  DR_REQUIRE(B >= 0 && num_buckets >= 1, DR_EINVAL, "%s: B=%lld num_buckets=%lld", who, (long long)B,
             (long long)num_buckets);
  DR_REQUIRE(values && value_offsets && row_splits && (out_splits || out_ids), DR_EINVAL, "%s: null pointer", who);
  ks->n = K;
  for (int i = 0; i < K; ++i) {
    DR_REQUIRE(values[i], DR_EINVAL, "%s: key %d has no values", who, i);
    DR_REQUIRE(out_splits || !row_splits[i], DR_EINVAL,
               "%s: key %d is multi-valued: the single-valued form (out_splits = NULL) cannot hold its crosses", who, i);
    ks->k[i] = cross::Key{values[i], value_offsets[i], row_splits[i]};
  }
  return DR_OK;
}
}  // namespace dr

extern "C" int dr_cross_hash(int K, const void* const* values, const int64_t* const* value_offsets,
                             const int64_t* const* row_splits, int64_t B, uint64_t hash_key, int64_t num_buckets,
                             int64_t* out_splits, int64_t* out_ids, void* stream) {
  cross::Keys ks;
  const int rc = cross_keys(K, values, value_offsets, row_splits, B, num_buckets, out_splits, out_ids,
                            "dr_cross_hash", &ks);
  if (rc != DR_OK) return rc;
  if (B == 0) return DR_OK;
  cross_hash_kernel<<<grid_for(B), 256, 0, (cudaStream_t)stream>>>(ks, B, hash_key, (uint64_t)num_buckets,
                                                                    out_splits, out_ids);
  DR_CUDA_LAUNCH_CHECK("dr_cross_hash");
  return DR_OK;
}

extern "C" int dr_cross_hash_host(int K, const void* const* values, const int64_t* const* value_offsets,
                                  const int64_t* const* row_splits, int64_t B, uint64_t hash_key, int64_t num_buckets,
                                  int64_t* out_splits, int64_t* out_ids) {
  cross::Keys ks;
  const int rc = cross_keys(K, values, value_offsets, row_splits, B, num_buckets, out_splits, out_ids,
                            "dr_cross_hash_host", &ks);
  if (rc != DR_OK) return rc;
  if (out_splits && !out_ids) out_splits[0] = 0;
  for (int64_t b = 0; b < B; ++b) {
    if (!out_splits) {
      if (cross::count(ks, b) == 1) cross::fill(ks, b, hash_key, (uint64_t)num_buckets, out_ids + b);
      else out_ids[b] = -1;
    } else if (!out_ids) {
      out_splits[b + 1] = cross::count(ks, b);
    } else {
      cross::fill(ks, b, hash_key, (uint64_t)num_buckets, out_ids + out_splits[b]);
    }
  }
  return DR_OK;
}
