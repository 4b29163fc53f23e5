// b2s_pit.cuh -- point-in-time (as-of) join of entity rows onto feature-set indexes: layouts and launch parameters shared
// by the sort and join kernels of b2s_pit.cu.
#pragma once
#include <cstdint>

#include "b2s_hash.cuh"

namespace b2s_pit {

// per launch: feature sets, their output columns, and entity columns permuted into sorted order (more are split over launches).
// One feature set per launch: on the H100, 4 sets x 32 features over 4 Mi entity rows joined in 7.6 ms as four launches
// against 9.5 ms as one launch looping over the sets (DESIGN.md §4g).
constexpr int kMaxSets = 1;
constexpr int kMaxOuts = 256;
constexpr int kMaxCols = 64;

struct OutCol {
  int32_t src_word;  // first 4-byte word of the column in the index's rows
  int32_t bytes;     // 4 or 8
  uint64_t miss;     // bits stored where the entity row has no match
  void* out;         // [n] elements
};

struct SetDesc {
  const b2s::TableSlot* slots;  // key -> (run start << 32 | run length)
  uint64_t mask;
  const int64_t* ts;            // [n_rows] feature-set timestamps, sorted by (key, ts)
  const uint32_t* rows;         // [n_rows][row_words] feature words in the same order
  int32_t row_words;
  int32_t asof;                 // 1: last row with ts <= the entity's ts; 0: the key's only row
  const int64_t* keys;          // [n] entity keys, input order
  int64_t* ts_out;              // [n] matched timestamp, INT64_MIN (NaT) on a miss; may be null
  uint8_t* found;               // [n] 1 / 0; may be null
  int32_t out0, n_out;          // outs[out0 .. out0 + n_out)
};

struct EntCol {
  const void* src;
  void* dst;
  int32_t bytes;  // 1, 2, 4 or 8
};

struct JoinParams {
  const int64_t* sorted_ts;       // [n] entity timestamps in sorted order; null when nothing is as-of
  const uint32_t* order;          // [n] input row at each sorted position; null: identity
  int64_t* order_out;             // [n] may be null
  int64_t q0, q1;                 // sorted positions this launch covers
  int32_t n_sets, n_cols;
  unsigned long long* miss;       // [n_sets] of this launch
  SetDesc sets[kMaxSets];
  OutCol outs[kMaxOuts];
  EntCol cols[kMaxCols];
};

}  // namespace b2s_pit
