// Device side of two contracts every scoring kernel keeps: where a row's label goes (LabelTargets), and the flag list
// of EXACT mode (FlagList) - the tile kernels append the rows they cannot certify, a re-score kernel reads them, counts
// them and hands the list back empty for the next launch on the stream.
#pragma once

#include "uml_common.cuh"

namespace uml {

// one row's label into every target: the local vector and each peer, int32 or uint8 (one lane)
__device__ __forceinline__ void store_label(const LabelTargets& t, long long row, int idx) {
  if (t.labels) t.labels[row] = idx;
  for (int i = 0; i < t.n_peers; ++i) {
    if (t.wire_u8) static_cast<uint8_t*>(t.peers[i])[t.row_offset + row] = static_cast<uint8_t>(idx);
    else static_cast<int32_t*>(t.peers[i])[t.row_offset + row] = idx;
  }
}

// a tile epilogue's store of one row: the local vector, and the peers when they are int32 (byte peers take whole words
// from store_label_word_u8)
__device__ __forceinline__ void store_label_i32(const LabelTargets& t, long long row, int idx) {
  if (t.labels) t.labels[row] = idx;
  if (!t.wire_u8)
    for (int i = 0; i < t.n_peers; ++i) static_cast<int32_t*>(t.peers[i])[t.row_offset + row] = idx;
}

// The helpers below take the kernel's parameter block `p` and read each field they need (targets, n_rows, flag_count,
// flag_rows, flag_cap, all_rows, counters) where they use it, as the kernels' own copies of this code did: with the
// fields read up front, or the destination computed after the lane test, ptxas schedules the tile kernels' epilogues
// differently.

// byte labels of rows row4 .. row4 + 3 (row row4 + b in byte b of `word`) into every peer of p.targets, from the lanes
// that hold a word (`active`): one aligned 4-byte store when all four rows are in the batch, all four are kept and the
// destination is word aligned, else one byte per kept row in the batch.  `keep` bit b clear: row row4 + b has another
// writer (a row the linear tensor-core schedule queued for its re-score warp), so its byte is not touched.
template <class P>
__device__ __forceinline__ void store_label_word_u8(const P& p, long long row4, uint32_t word, bool active,
                                                    unsigned keep = 0xfu) {
  const long long at = p.targets.row_offset + row4;
  if (active) {
    if (keep == 0xfu && row4 + 3 < p.n_rows && (at & 3) == 0) {
      for (int i = 0; i < p.targets.n_peers; ++i) *reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(p.targets.peers[i]) + at) = word;
    } else {
      for (int b = 0; b < 4; ++b)
        if (((keep >> b) & 1u) && row4 + b < p.n_rows)
          for (int i = 0; i < p.targets.n_peers; ++i)
            static_cast<uint8_t*>(p.targets.peers[i])[at + b] = static_cast<uint8_t>((word >> (8 * b)) & 0xffu);
    }
  }
}

// the flagged rows of a warp (at most one per lane) onto the flag list with one atomic; entries past flag_cap are
// dropped (the re-score reads min(count, cap) of them)
template <class P>
__device__ __forceinline__ void flag_rows_warp(bool flagged, long long row, const P& p, int lane) {
  const unsigned mask = __ballot_sync(0xffffffffu, flagged);
  if (mask != 0u) {
    int base = 0;
    if (lane == 0) base = atomicAdd(p.flag_count, __popc(mask));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (flagged) {
      const int pos = base + __popc(mask & ((1u << lane) - 1u));
      if (pos < p.flag_cap) p.flag_rows[pos] = static_cast<int32_t>(row);
    }
  }
}

// the number of rows a re-score launch scores: every row of the batch, or the flag list's entries, which count once
// per launch into kCounterFlagged
template <class P>
__device__ __forceinline__ long long flag_list_rows(const P& p) {
  const long long n = p.all_rows ? p.n_rows : static_cast<long long>(min(*p.flag_count, p.flag_cap));
  if (!p.all_rows && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&p.counters[kCounterFlagged], static_cast<unsigned long long>(n));
  return n;
}

// the end of a re-score launch (every thread): every block has read *flag_count before it gets here, so the last one
// to finish may reset it and the ticket for the next scoring launch on the stream - no memset between steps
template <class P>
__device__ __forceinline__ void flag_list_hand_back(const P& p) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned long long ticket = atomicAdd(&p.counters[kCounterRescoreTicket], 1ull);
    if (ticket == static_cast<unsigned long long>(gridDim.x) - 1ull) {
      *const_cast<int*>(p.flag_count) = 0;
      p.counters[kCounterRescoreTicket] = 0ull;
      __threadfence();
    }
  }
}

// a re-scored row's outcome into the launch's counters (one lane)
template <class P>
__device__ __forceinline__ void count_rescored_row(const P& p, bool bad, bool ambiguous) {
  if (bad) atomicAdd(&p.counters[kCounterNonfinite], 1ull);
  if (ambiguous) atomicAdd(&p.counters[kCounterAmbiguous], 1ull);
}

}  // namespace uml
