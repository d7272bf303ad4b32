// SURVEY.md 8(f) #4 -- the input format in front of the id pipeline: `movielens.tfrecords`, a TFRecord file of
// serialized tf.train.Example protos (writer schema datasets/movielens.py:54-62, reader :116-125:
// FixedLenFeature int64 / string per column, VarLenFeature string for "Genres").  In the reference both the record
// framing and the proto parse are TensorFlow's C++ (tf.data.TFRecordDataset, tf.io.parse_example); here they are
// host entry points of the same C-ABI library, so a batch goes  file bytes -> columnar (values | packed strings +
// offsets | row_splits) -> dr_hash_bucket_bytes_host / dr_vocab_lookup_* -> int64 ids  without a Python loop.
// Host-only code (no kernels): the formats are byte-exact public formats, restated from their specifications:
//   TFRecord framing   uint64 length | uint32 masked_crc32c(length) | data | uint32 masked_crc32c(data), little endian,
//                      mask(c) = rotr(c, 15) + 0xa282ead8
//   CRC-32C            Castagnoli polynomial 0x1EDC6F41 (reflected 0x82F63B78), RFC 3720 appendix B.4 test vectors
//   Example            protobuf wire format: Example{1: Features{1: map<string, Feature>}},
//                      Feature{1: BytesList | 2: FloatList | 3: Int64List}, lists{1: repeated value}, scalars packed
//                      or unpacked.
#include <string.h>
#include <atomic>
#include <mutex>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <vector>
#include "common.cuh"

namespace dr {
namespace tfr {

static uint32_t g_crc_table[8][256];
static std::once_flag g_crc_once;

static void crc_fill() {
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
    g_crc_table[0][i] = c;
  }
  for (uint32_t i = 0; i < 256; ++i)
    for (int t = 1; t < 8; ++t) g_crc_table[t][i] = (g_crc_table[t - 1][i] >> 8) ^ g_crc_table[0][g_crc_table[t - 1][i] & 0xff];
}
// ctypes releases the GIL: two host threads may open files concurrently, so the table is built exactly once
static void crc_init() { std::call_once(g_crc_once, crc_fill); }

static uint32_t crc32c(const uint8_t* p, size_t n) {
  crc_init();
  uint32_t c = 0xffffffffu;
  while (n >= 8) {   // slicing-by-8
    uint64_t w;
    memcpy(&w, p, 8);
    w ^= c;
    c = g_crc_table[7][w & 0xff] ^ g_crc_table[6][(w >> 8) & 0xff] ^ g_crc_table[5][(w >> 16) & 0xff] ^
        g_crc_table[4][(w >> 24) & 0xff] ^ g_crc_table[3][(w >> 32) & 0xff] ^ g_crc_table[2][(w >> 40) & 0xff] ^
        g_crc_table[1][(w >> 48) & 0xff] ^ g_crc_table[0][(w >> 56) & 0xff];
    p += 8;
    n -= 8;
  }
  while (n--) c = (c >> 8) ^ g_crc_table[0][(c ^ *p++) & 0xff];
  return c ^ 0xffffffffu;
}

static inline uint32_t mask_crc(uint32_t c) { return ((c >> 15) | (c << 17)) + 0xa282ead8u; }

// ---- protobuf wire helpers ------------------------------------------------------------------------------------
struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  bool more() const { return ok && p < end; }
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p >= end) { ok = false; return 0; }
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  Cursor sub() {   // length-delimited payload
    const uint64_t n = varint();
    if (!ok || n > (uint64_t)(end - p)) { ok = false; return Cursor{p, p, false}; }
    Cursor c{p, p + n, true};
    p += n;
    return c;
  }
  void skip(int wire) {
    switch (wire) {
      case 0: varint(); break;
      case 1: if (end - p < 8) ok = false; else p += 8; break;
      case 2: sub(); break;
      case 5: if (end - p < 4) ok = false; else p += 4; break;
      default: ok = false;
    }
  }
};

// Finds Feature `name` inside one serialized Example; returns its payload cursor (ok == false: malformed; empty
// range with found == false: the feature is absent).
static Cursor find_feature(const uint8_t* rec, int64_t len, const char* name, size_t name_len, bool* found) {
  *found = false;
  Cursor ex{rec, rec + len, true};
  Cursor result{rec, rec, true};
  while (ex.more()) {
    const uint64_t tag = ex.varint();
    if (!ex.ok) break;
    if ((tag >> 3) == 1 && (tag & 7) == 2) {          // Example.features
      Cursor feats = ex.sub();
      while (feats.more()) {
        const uint64_t t2 = feats.varint();
        if (!feats.ok) break;
        if ((t2 >> 3) == 1 && (t2 & 7) == 2) {        // Features.feature map entry
          Cursor entry = feats.sub();
          bool key_match = false;
          Cursor value{entry.p, entry.p, true};
          bool has_value = false;
          while (entry.more()) {
            const uint64_t t3 = entry.varint();
            if (!entry.ok) break;
            if ((t3 >> 3) == 1 && (t3 & 7) == 2) {
              Cursor key = entry.sub();
              key_match = key.ok && (size_t)(key.end - key.p) == name_len && memcmp(key.p, name, name_len) == 0;
            } else if ((t3 >> 3) == 2 && (t3 & 7) == 2) {
              value = entry.sub();
              has_value = true;
            } else {
              entry.skip((int)(t3 & 7));
            }
          }
          if (!entry.ok) { result.ok = false; return result; }
          if (key_match) {       // later duplicates of a map key win (protobuf map semantics)
            *found = true;
            result = has_value ? value : Cursor{entry.end, entry.end, true};
          }
        } else {
          feats.skip((int)(t2 & 7));
        }
      }
      if (!feats.ok) { result.ok = false; return result; }
    } else {
      ex.skip((int)(tag & 7));
    }
  }
  if (!ex.ok) result.ok = false;
  return result;
}

enum { KIND_INT64 = 0, KIND_BYTES = 1, KIND_FLOAT = 2 };

// Walks the values of one Feature payload.  on_scalar(bits) for int64 / float, on_bytes(ptr, len) for bytes.
// Returns false on malformed input or a kind mismatch (a feature stored as another list type).
template <typename FS, typename FB>
static bool walk_values(Cursor feat, int kind, FS on_scalar, FB on_bytes) {
  const uint64_t want_field = kind == KIND_BYTES ? 1 : (kind == KIND_FLOAT ? 2 : 3);
  while (feat.more()) {
    const uint64_t tag = feat.varint();
    if (!feat.ok) return false;
    if ((tag & 7) != 2) { feat.skip((int)(tag & 7)); continue; }
    Cursor list = feat.sub();
    if (!feat.ok) return false;
    if ((tag >> 3) != want_field) {
      if ((tag >> 3) >= 1 && (tag >> 3) <= 3 && list.p != list.end) return false;   // another, non-empty list kind
      continue;
    }
    while (list.more()) {
      const uint64_t t = list.varint();
      if (!list.ok || (t >> 3) != 1) return false;
      const int wire = (int)(t & 7);
      if (kind == KIND_BYTES) {
        if (wire != 2) return false;
        Cursor b = list.sub();
        if (!list.ok) return false;
        on_bytes(b.p, (int64_t)(b.end - b.p));
      } else if (kind == KIND_INT64) {
        if (wire == 2) {          // packed
          Cursor pk = list.sub();
          if (!list.ok) return false;
          while (pk.more()) { const uint64_t v = pk.varint(); if (!pk.ok) return false; on_scalar(v); }
        } else if (wire == 0) {
          const uint64_t v = list.varint();
          if (!list.ok) return false;
          on_scalar(v);
        } else return false;
      } else {
        if (wire == 2) {
          Cursor pk = list.sub();
          if (!list.ok || ((pk.end - pk.p) & 3)) return false;
          for (; pk.p < pk.end; pk.p += 4) { uint32_t v; memcpy(&v, pk.p, 4); on_scalar((uint64_t)v); }
        } else if (wire == 5) {
          if (list.end - list.p < 4) return false;
          uint32_t v; memcpy(&v, list.p, 4); list.p += 4;
          on_scalar((uint64_t)v);
        } else return false;
      }
    }
    if (!list.ok) return false;
  }
  return feat.ok;
}

}  // namespace tfr
}  // namespace dr

using namespace dr;

extern "C" uint32_t dr_crc32c_host(const uint8_t* data, int64_t n) { return tfr::crc32c(data, n < 0 ? 0 : (size_t)n); }
extern "C" uint32_t dr_masked_crc32c_host(const uint8_t* data, int64_t n) {
  return tfr::mask_crc(tfr::crc32c(data, n < 0 ? 0 : (size_t)n));
}

extern "C" int64_t dr_tfrecord_index(const uint8_t* buf, int64_t nbytes, int verify_crc, int64_t* rec_off,
                                     int64_t* rec_len, int64_t cap) {
  DR_REQUIRE(nbytes >= 0 && (buf || nbytes == 0), DR_EINVAL, "dr_tfrecord_index: null buffer");
  int64_t pos = 0, n = 0;
  while (pos < nbytes) {
    DR_REQUIRE(nbytes - pos >= 12, DR_EINVAL, "dr_tfrecord_index: truncated record header at byte %lld", (long long)pos);
    uint64_t len;
    uint32_t crc;
    memcpy(&len, buf + pos, 8);
    memcpy(&crc, buf + pos + 8, 4);
    if (verify_crc)
      DR_REQUIRE(tfr::mask_crc(tfr::crc32c(buf + pos, 8)) == crc, DR_EINVAL,
                 "dr_tfrecord_index: corrupted record length at byte %lld (crc mismatch)", (long long)pos);
    DR_REQUIRE(len <= (uint64_t)(nbytes - pos - 12) && (uint64_t)(nbytes - pos - 12) - len >= 4, DR_EINVAL,
               "dr_tfrecord_index: truncated record %lld (length %llu)", (long long)n, (unsigned long long)len);
    if (verify_crc) {
      memcpy(&crc, buf + pos + 12 + len, 4);
      DR_REQUIRE(tfr::mask_crc(tfr::crc32c(buf + pos + 12, (size_t)len)) == crc, DR_EINVAL,
                 "dr_tfrecord_index: corrupted record %lld at byte %lld (crc mismatch)", (long long)n, (long long)pos);
    }
    if (rec_off && n < cap) rec_off[n] = pos + 12;
    if (rec_len && n < cap) rec_len[n] = (int64_t)len;
    ++n;
    pos += 12 + (int64_t)len + 4;
  }
  return n;
}

// One feature of `n` serialized Examples -> columnar.  Call once with values == bytes == NULL to size the outputs
// (row_splits, *total_values, *total_bytes are filled), then again with buffers of at least that size.
extern "C" int dr_example_parse_feature(const uint8_t* buf, const int64_t* rec_off, const int64_t* rec_len, int64_t n,
                                        const char* name, int kind, int64_t* row_splits, void* values,
                                        uint8_t* bytes, int64_t* value_offsets, int64_t* total_values,
                                        int64_t* total_bytes) {
  DR_REQUIRE(n >= 0 && name && (n == 0 || (buf && rec_off && rec_len)), DR_EINVAL, "dr_example_parse_feature: null pointer");
  DR_REQUIRE(kind >= 0 && kind <= 2, DR_EINVAL, "dr_example_parse_feature: kind=%d (0 int64, 1 bytes, 2 float)", kind);
  const size_t name_len = strlen(name);
  int64_t nv = 0, nb = 0;
  if (row_splits) row_splits[0] = 0;
  if (value_offsets) value_offsets[0] = 0;
  for (int64_t r = 0; r < n; ++r) {
    bool found = false;
    tfr::Cursor feat = tfr::find_feature(buf + rec_off[r], rec_len[r], name, name_len, &found);
    DR_REQUIRE(feat.ok, DR_EINVAL, "dr_example_parse_feature: record %lld is not a valid tf.train.Example", (long long)r);
    if (found) {
      const bool ok = tfr::walk_values(
          feat, kind,
          [&](uint64_t bits) {
            if (values) {
              if (kind == tfr::KIND_INT64) reinterpret_cast<int64_t*>(values)[nv] = (int64_t)bits;
              else { const uint32_t b32 = (uint32_t)bits; memcpy(reinterpret_cast<float*>(values) + nv, &b32, 4); }
            }
            ++nv;
          },
          [&](const uint8_t* p, int64_t len) {
            if (bytes) memcpy(bytes + nb, p, (size_t)len);
            nb += len;
            ++nv;
            if (value_offsets) value_offsets[nv] = nb;
          });
      DR_REQUIRE(ok, DR_EINVAL, "dr_example_parse_feature: feature '%s' of record %lld is malformed or not of the requested kind",
                 name, (long long)r);
    }
    if (row_splits) row_splits[r + 1] = nv;
  }
  if (total_values) *total_values = nv;
  if (total_bytes) *total_bytes = nb;
  return DR_OK;
}

// All requested features of n records in ONE walk per record (the single-feature entry above walks a record once per
// feature).  Same two-pass protocol: with values == NULL (or all its entries NULL) only row_splits[f][0..n],
// total_values[f] and total_bytes[f] are written; then the caller allocates and calls again.
// Large batches CAN be parsed by several host threads (dr_set_host_threads; tf.data's num_parallel_calls): record
// ranges are counted in parallel, a serial prefix over the ranges gives every range its output offsets, then the
// ranges are filled in parallel -- the output is identical for any thread count.  The threaded path walks every
// record three times instead of two; it pays only when the output buffers are already faulted in (first-touch page
// faults of fresh buffers dominate otherwise; tools/bench_tfrecord.py times both), so serial is the default and
// threading is opt-in.
namespace dr {
namespace tfr {

static std::atomic<int> g_host_threads{1};   // 1 = serial (default); 0 = min(hardware threads, 8)

struct BatchCtx {
  const uint8_t* buf;
  const int64_t* rec_off;
  const int64_t* rec_len;
  int nfeat;
  const char* const* names;
  const size_t* name_len;
  const int* kinds;
  int64_t* const* row_splits;
  void* const* values;
  uint8_t* const* bytes;
  int64_t* const* value_offsets;
};

// Walks records [r0, r1).  nv / nb: running value / byte counters per feature (in: start, out: end).
// write_splits: row_splits[f][r + 1] = nv[f] after every record.  fill: write values / bytes / value_offsets.
// Returns DR_OK or DR_EINVAL with *err_rec / err describing the first bad record of the range.
static int walk_records(const BatchCtx& c, int64_t r0, int64_t r1, int64_t* nv, int64_t* nb, bool write_splits,
                        bool fill, int64_t* err_rec, std::string* err) {
  int64_t nv0[256], nb0[256];
  for (int64_t r = r0; r < r1; ++r) {
    for (int f = 0; f < c.nfeat; ++f) { nv0[f] = nv[f]; nb0[f] = nb[f]; }
    Cursor ex{c.buf + c.rec_off[r], c.buf + c.rec_off[r] + c.rec_len[r], true};
    bool bad = false;
    while (ex.more() && !bad) {
      const uint64_t tag = ex.varint();
      if (!ex.ok) break;
      if ((tag >> 3) != 1 || (tag & 7) != 2) { ex.skip((int)(tag & 7)); continue; }
      Cursor feats = ex.sub();                            // Example.features
      while (feats.more() && !bad) {
        const uint64_t t2 = feats.varint();
        if (!feats.ok) break;
        if ((t2 >> 3) != 1 || (t2 & 7) != 2) { feats.skip((int)(t2 & 7)); continue; }
        Cursor entry = feats.sub();                       // map entry {1: key, 2: Feature}
        int f = -1;
        Cursor value{entry.p, entry.p, true};
        while (entry.more()) {
          const uint64_t t3 = entry.varint();
          if (!entry.ok) break;
          if ((t3 >> 3) == 1 && (t3 & 7) == 2) {
            Cursor key = entry.sub();
            const size_t kl = key.ok ? (size_t)(key.end - key.p) : 0;
            f = -1;
            for (int g = 0; g < c.nfeat; ++g)
              if (kl == c.name_len[g] && memcmp(key.p, c.names[g], kl) == 0) { f = g; break; }
          } else if ((t3 >> 3) == 2 && (t3 & 7) == 2) {
            value = entry.sub();
          } else {
            entry.skip((int)(t3 & 7));
          }
        }
        if (!entry.ok) { bad = true; break; }
        if (f < 0) continue;
        nv[f] = nv0[f];                                   // a repeated map key: the later entry wins
        nb[f] = nb0[f];
        void* vals = (fill && c.values) ? c.values[f] : nullptr;
        uint8_t* by = (fill && c.bytes) ? c.bytes[f] : nullptr;
        int64_t* vo = (fill && c.value_offsets) ? c.value_offsets[f] : nullptr;
        const int kind = c.kinds[f];
        const bool ok = walk_values(
            value, kind,
            [&](uint64_t bits) {
              if (vals) {
                if (kind == KIND_INT64) reinterpret_cast<int64_t*>(vals)[nv[f]] = (int64_t)bits;
                else { const uint32_t b32 = (uint32_t)bits; memcpy(reinterpret_cast<float*>(vals) + nv[f], &b32, 4); }
              }
              ++nv[f];
            },
            [&](const uint8_t* p, int64_t len) {
              if (by) memcpy(by + nb[f], p, (size_t)len);
              nb[f] += len;
              ++nv[f];
              if (vo) vo[nv[f]] = nb[f];
            });
        if (!ok) {
          *err_rec = r;
          *err = std::string("feature '") + c.names[f] + "' of record " + std::to_string((long long)r) +
                 " is malformed or not of the requested kind";
          return DR_EINVAL;
        }
      }
      if (!feats.ok) bad = true;
    }
    if (bad || !ex.ok) {
      *err_rec = r;
      *err = "record " + std::to_string((long long)r) + " is not a valid tf.train.Example";
      return DR_EINVAL;
    }
    if (write_splits)
      for (int f = 0; f < c.nfeat; ++f) c.row_splits[f][r + 1] = nv[f];
  }
  return DR_OK;
}

}  // namespace tfr
}  // namespace dr

extern "C" int dr_set_host_threads(int n) {
  DR_REQUIRE(n >= 0 && n <= 256, DR_EINVAL, "dr_set_host_threads: n=%d outside [0, 256]", n);
  tfr::g_host_threads = n;
  return DR_OK;
}

extern "C" int dr_example_parse_batch(const uint8_t* buf, const int64_t* rec_off, const int64_t* rec_len, int64_t n,
                                      int nfeat, const char* const* names, const int* kinds,
                                      int64_t* const* row_splits, void* const* values, uint8_t* const* bytes,
                                      int64_t* const* value_offsets, int64_t* total_values, int64_t* total_bytes) {
  DR_REQUIRE(n >= 0 && nfeat >= 1 && nfeat <= 256 && names && kinds && row_splits && total_values && total_bytes,
             DR_EINVAL, "dr_example_parse_batch: bad arguments (n=%lld nfeat=%d)", (long long)n, nfeat);
  DR_REQUIRE(n == 0 || (buf && rec_off && rec_len), DR_EINVAL, "dr_example_parse_batch: null record index");
  size_t name_len[256];
  bool fill = false;
  for (int f = 0; f < nfeat; ++f) {
    DR_REQUIRE(names[f] && kinds[f] >= 0 && kinds[f] <= 2 && row_splits[f], DR_EINVAL,
               "dr_example_parse_batch: feature %d: null name / row_splits or kind outside 0..2", f);
    name_len[f] = strlen(names[f]);
    row_splits[f][0] = 0;
    if (value_offsets && value_offsets[f]) value_offsets[f][0] = 0;
    fill = fill || (values && values[f]) || (bytes && bytes[f]);
  }
  const tfr::BatchCtx c{buf, rec_off, rec_len, nfeat, names, name_len, kinds, row_splits, values, bytes, value_offsets};
  int T = tfr::g_host_threads;
  if (T == 0) {
    const unsigned hw = std::thread::hardware_concurrency();
    T = hw == 0 ? 1 : (hw > 8 ? 8 : (int)hw);
  }
  if ((int64_t)T > n / 2048) T = (int)(n / 2048);       // at least 2048 records per thread
  if (T <= 1) {
    int64_t nv[256] = {0}, nb[256] = {0}, er = -1;
    std::string err;
    if (tfr::walk_records(c, 0, n, nv, nb, true, fill, &er, &err) != DR_OK) {
      set_error("dr_example_parse_batch: %s", err.c_str());
      return DR_EINVAL;
    }
    for (int f = 0; f < nfeat; ++f) { total_values[f] = nv[f]; total_bytes[f] = nb[f]; }
    return DR_OK;
  }
  // ---- threaded: count per range -> prefix over ranges -> fix row_splits up (and fill) per range ----------------
  std::vector<int64_t> cnt_v((size_t)T * nfeat, 0), cnt_b((size_t)T * nfeat, 0), err_rec((size_t)T, -1);
  std::vector<int> rc((size_t)T, DR_OK);
  std::vector<std::string> errs((size_t)T);
  auto range = [&](int t, int64_t* r0, int64_t* r1) { *r0 = n * t / T; *r1 = n * (t + 1) / T; };
  auto run = [&](auto&& fn) {
    std::vector<std::thread> th;
    for (int t = 1; t < T; ++t) th.emplace_back(fn, t);
    fn(0);
    for (auto& x : th) x.join();
  };
  auto first_error = [&]() -> int {
    int best = -1;
    for (int t = 0; t < T; ++t)
      if (rc[t] != DR_OK && (best < 0 || err_rec[t] < err_rec[best])) best = t;
    if (best < 0) return DR_OK;
    set_error("dr_example_parse_batch: %s", errs[best].c_str());
    return DR_EINVAL;
  };
  run([&](int t) {
    int64_t r0, r1;
    range(t, &r0, &r1);
    int64_t nv[256] = {0}, nb[256] = {0}, er = -1;      // counters on this thread's stack (no false sharing)
    std::string err;
    rc[t] = tfr::walk_records(c, r0, r1, nv, nb, true, false, &er, &err);   // row_splits relative to the range start for now
    for (int f = 0; f < nfeat; ++f) { cnt_v[(size_t)t * nfeat + f] = nv[f]; cnt_b[(size_t)t * nfeat + f] = nb[f]; }
    err_rec[t] = er;
    errs[t] = err;
  });
  if (int e = first_error()) return e;
  std::vector<int64_t> base_v((size_t)T * nfeat, 0), base_b((size_t)T * nfeat, 0);
  for (int f = 0; f < nfeat; ++f) {
    int64_t av = 0, ab = 0;
    for (int t = 0; t < T; ++t) {
      base_v[(size_t)t * nfeat + f] = av;
      base_b[(size_t)t * nfeat + f] = ab;
      av += cnt_v[(size_t)t * nfeat + f];
      ab += cnt_b[(size_t)t * nfeat + f];
    }
    total_values[f] = av;
    total_bytes[f] = ab;
  }
  run([&](int t) {
    int64_t r0, r1;
    range(t, &r0, &r1);
    for (int f = 0; f < nfeat; ++f) {
      const int64_t add = base_v[(size_t)t * nfeat + f];
      if (add)
        for (int64_t r = r0; r < r1; ++r) row_splits[f][r + 1] += add;
    }
    if (fill) {
      int64_t nv[256], nb[256];
      for (int f = 0; f < nfeat; ++f) { nv[f] = base_v[(size_t)t * nfeat + f]; nb[f] = base_b[(size_t)t * nfeat + f]; }
      int64_t er = -1;
      std::string err;
      rc[t] = tfr::walk_records(c, r0, r1, nv, nb, false, true, &er, &err);
      err_rec[t] = er;
      errs[t] = err;
    }
  });
  return first_error();
}

// categorical_column_with_vocabulary_list on string keys: position in the list, out-of-vocabulary -> default_id.
extern "C" int dr_vocab_lookup_bytes_host(const uint8_t* bytes, const int64_t* offsets, int64_t n,
                                          const uint8_t* vocab_bytes, const int64_t* vocab_offsets, int64_t vocab_size,
                                          int64_t default_id, int64_t* out_ids) {
  DR_REQUIRE(n >= 0 && vocab_size >= 0, DR_EINVAL, "dr_vocab_lookup_bytes_host: n=%lld vocab_size=%lld", (long long)n,
             (long long)vocab_size);
  if (n == 0) return DR_OK;
  DR_REQUIRE(offsets && out_ids && (vocab_offsets || vocab_size == 0), DR_EINVAL, "dr_vocab_lookup_bytes_host: null pointer");
  std::unordered_map<std::string_view, int64_t> table;
  table.reserve((size_t)vocab_size * 2);
  for (int64_t i = 0; i < vocab_size; ++i)   // first occurrence wins (TF rejects duplicate vocabulary entries)
    table.emplace(std::string_view(reinterpret_cast<const char*>(vocab_bytes) + vocab_offsets[i],
                                   (size_t)(vocab_offsets[i + 1] - vocab_offsets[i])), i);
  for (int64_t i = 0; i < n; ++i) {
    DR_REQUIRE(offsets[i + 1] >= offsets[i], DR_EINVAL, "dr_vocab_lookup_bytes_host: offsets not monotone at %lld", (long long)i);
    auto it = table.find(std::string_view(reinterpret_cast<const char*>(bytes) + offsets[i], (size_t)(offsets[i + 1] - offsets[i])));
    out_ids[i] = it == table.end() ? default_id : it->second;
  }
  return DR_OK;
}
