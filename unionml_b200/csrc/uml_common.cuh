// Shared declarations for the uml_b200 CUDA library (sm_90a only).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/uml_b200.h"

namespace uml {

// ---------------------------------------------------------------------------------------------------------------
// Tile geometry of the TMA fp32 scoring kernel (see DESIGN.md "linear_argmax_tma")
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTileRows = 128;                            // rows per stage = TMA box height
constexpr int kChunkF = 32;                               // features per stage = TMA box width (128 B -> SWIZZLE_128B)
constexpr int kStageBytes = kTileRows * kChunkF * 4;      // 16 KiB
constexpr int kConsumerWarps = 8;                         // 2 per SM sub-partition
constexpr int kThreads = (kConsumerWarps + 1) * 32;       // + 1 TMA producer warp
constexpr int kRowsPerLane = kTileRows / 32;              // R = 4 rows per thread
constexpr int kMaxClassesTma = 16;                        // classes handled in registers by the TMA kernel
constexpr int kMaxSmemBytes = 227 * 1024;
// Whole-row schedule of the linear tile kernel (33 <= F <= 64, f_pad = 64): one stage holds complete rows, 64 rows x
// 64 features = kStageBytes, loaded as two {32, 64} boxes onto one barrier.  Other widths keep 128-row boxes: at
// F <= 32 one box already holds whole rows, and wider rows do not fit eight stages.
constexpr int kWholeTileRows = kStageBytes / (2 * kChunkF * 4);  // 64
__host__ __device__ inline bool linear_whole_rows(int f_pad) { return f_pad == 2 * kChunkF; }
// rows per box of the tensor map the linear tile kernel reads (its feature width is always kChunkF)
__host__ __device__ inline int linear_box_rows(int f_pad) { return linear_whole_rows(f_pad) ? kWholeTileRows : kTileRows; }
// Compact fp16 rows (F <= 64, every value an fp16 value): one {64 features, 128 rows} fp16 box = 128 whole rows in
// kStageBytes, read through the batch's half_map
constexpr int kHalfBoxF = 2 * kChunkF;  // 64 halves = 128 bytes per row, the SWIZZLE_128B span
__host__ __device__ inline bool linear_half_rows_ok(int f_pad) { return f_pad <= kHalfBoxF; }
__host__ __device__ inline int linear_half_ld(int F) { return (F + 7) / 8 * 8; }  // halves per row: 16-byte row pitch
// Ring items of the fp16 schedule: 256 whole rows, two {64, 128} fp16 boxes on one barrier (32 KiB), so a lane scores
// 8 rows and every broadcast W load feeds 8 FMA chains per class instead of 4.  Its feed outruns the scoring warps
// (their cost per row is the limit, DESIGN.md 5.1).
constexpr int kHalfTileRows = 2 * kTileRows;
// Scoring warps of the fp16 schedule: one per SM sub-partition, with up to 255 registers for its 8 rows of
// accumulators and the operands of the next feature.  The ring must hold at least this many items.
constexpr int kHalfConsumerWarps = 4;
// Byte rows (F <= 64, every value an integer in [0, 255]): 64 bytes per row, zeros past F, one {64, 256} uint8 box =
// one 256-row ring item of kStageBytes.  The bytes of a row are stored in the order of the f16 A fragment of wgmma
// m64nNk16 (PTX ISA, "Register fragments, A, .f16"): the thread of column group t = lane % 4 loads the 16 bytes at
// 16 t, and their word s holds the four features it owns in k16 step s, 16 s + {2t, 2t+1, 2t+8, 2t+9}.
constexpr int kByteRowBytes = 64;
__host__ __device__ inline int linear_byte_pos(int f) {
  return 16 * ((f & 7) >> 1) + 4 * (f >> 4) + 2 * ((f >> 3) & 1) + (f & 1);
}

struct LinearDeviceModel {
  // fp32 operands of the tile kernel: wt[f][cp] (feature-major, classes padded to cp = 4*ceil((C+1)/4), column C holds
  // wmax_f = max_c |w_cf| for the error bound), bias[cp] (column C = max_c |b_c|)
  const float* wt;
  const float* bias;
  // fp64 operands of the re-score / generic kernel: w64[F][w64_stride] (feature-major, classes contiguous and zero
  // padded; see linear_w64_stride), b64[2C] = the biases, then each class's bias magnitude for the error bound
  const double* w64;
  const double* b64;
  int w64_stride;
  double fold_rel;  // extra relative term of the fp64 bound for a folded affine map (DESIGN.md 3.2), else 0
  int binary;       // the caller's model has one coef_ row: sklearn's `score > 0` rule, NaN gives class 0
  int n_classes;   // C after binary expansion (>= 2)
  int n_features;  // F
  int cp;          // padded class columns in wt
  int f_pad;       // rows of wt = 32 * ceil(F / 32), zero padded
  // tensor-core schedule of the fp16 rows (DESIGN.md 3.1, 3.2), nullptr when the model does not qualify: the B operand
  // [n][64] fp16, n = linear_tc_cols(C), W^T scaled by 2^sigma as hi | lo pieces with the bound column at hi column C,
  // pre-swizzled (SWIZZLE_128B, one 128-byte row per column) so one linear copy fills shared memory; then the scaled
  // biases as fp32 at byte n * 128 (hi columns: b_c for c < C, the bound column's bias at C, 0 past it)
  const void* tc_ops;
  float tc_kappa;  // a row is certain iff margin > tc_kappa * A (scaled scores, DESIGN.md 3.2)
};
// hi and lo column blocks of the tensor-core B operand: the C classes and the bound column, then the C lo pieces, each
// padded to a multiple of 8 so that a class's hi and lo accumulators sit in the same thread of the wgmma fragment
__host__ __device__ constexpr int linear_tc_hi_cols(int C) { return (C + 1 + 7) / 8 * 8; }
__host__ __device__ constexpr int linear_tc_cols(int C) { return linear_tc_hi_cols(C) + (C + 7) / 8 * 8; }

// doubles per feature of the fp64 weight table: a lane reads the classes of ITS feature as 16-byte pairs, so the row
// length in 16-byte units must be odd for the eight lanes of a quarter-warp to land in eight different bank groups of
// shared memory (C = 10 -> 10 doubles = 80 bytes, C = 16 -> 18, C = 2 -> 2); rounds of 16 classes stay 16-byte aligned
__host__ __device__ inline int linear_w64_stride(int n_classes) {
  int pairs = (n_classes + 1) / 2;
  if (pairs % 2 == 0) pairs += 1;
  return 2 * pairs;
}

// ---------------------------------------------------------------------------------------------------------------
// Exactness bounds below FLT_MIN (DESIGN.md 3.2-3.4).  The margin guards compare fp32 margins with a RELATIVE bound
// (a multiple of u = 2^-24 times an accumulated |.| sum); an fp32 rounding whose result is subnormal errs by up to
// 2^-150 absolute instead, and a tensor-core flush by up to FLT_MIN.  These host-side constants make the bound columns
// cover that: they are ~1e-37 of A on ordinary data, so they round away there and change no flag decision.  The bound
// entries are rounded to nearest; that relative error (u) is inside the 1.0001 slack of every threshold.
// ---------------------------------------------------------------------------------------------------------------
constexpr double kU = 5.9604644775390625e-08;            // 2^-24
constexpr double kFltMin = 1.1754943508222875e-38;       // 2^-126
constexpr double kHalfSubnormal = 7.006492321624085e-46;  // 2^-150: largest error of a rounding into the subnormals
// linear tile kernel: a row is certain iff margin > thr * A, thr = 2 err / A, err <= (F+4) u A (1 + F 2^-21)
inline float linear_margin_thr(int F) {
  return static_cast<float>(2.0 * (F + 4.0) * kU * (1.0 + F * 4.76837158203125e-07) * 1.0001);
}
// MLP kernels: the layer-2 term of err = e1 A1 + e2 A2
inline float mlp_e2_scale(int H) { return static_cast<float>((H + 4.0) * kU * 1.0001); }
// entry C of the A2 bias column: max_c |b2_c| plus K2 with e2 K2 >= FLT_MIN + (absolute error of a logit), where a
// hidden unit carries at most `hidden_abs` absolute error into layer 2 (weighted by max_c sum_n |w2_cn|) and the H
// fp32 FMAs of layer 2, the two bias adds and the two products of err add 2^-150 each.  The FLT_MIN keeps e2 A2
// (and so err) a normal number, where the comparison with the margin is relative again.
inline float mlp_a2_bias_entry(float b2max, double hidden_abs, double w2_abs_row_sum_max, int H) {
  const double babs = hidden_abs * w2_abs_row_sum_max + (H + 4.0) * kHalfSubnormal;
  return static_cast<float>(static_cast<double>(b2max) + (kFltMin + babs) / mlp_e2_scale(H) * (1.0 + 1.0 / 1024));
}

struct FlagList {
  int* count;        // number of flagged rows appended so far; the re-score kernel's last block resets it to 0
  int32_t* rows;     // flagged row indices
  int capacity;
  unsigned long long* counters;  // [kCounterSlots]
};
// slots of FlagList::counters.  A synchronous call zeroes those before kCounterTileClaim and reads them back; the
// re-score kernels hand the ticket back at 0, the linear tile kernel both claim slots, so a step needs no memset.
enum Counter : int {
  kCounterAmbiguous,      // rows whose float64 margin is inside its rounding bound (uml_stats.n_ambiguous)
  kCounterNonfinite,      // rows with NaN / Inf (n_nonfinite)
  kCounterFlagged,        // rows re-scored in float64 (n_flagged)
  kCounterRescoreTicket,  // re-score blocks done; the last one hands the flag list back empty (label_store.cuh)
  kCounterTileClaim,      // the linear tile kernel's next unclaimed tile
  kCounterTileClaimDone,  // its CTAs done claiming; the last one hands both claim slots back at 0
  kCounterSlots
};

// The caller's own values for the rows of a launch: the raw source chunk as it was copied to the device (any dtype,
// either memory order).  The fp64 re-score reads the flagged rows from here, so labels follow the float64 (or int64)
// features the caller passed even when their fp32 copy is lossy (sklearn scores the float64 frame, _base.py:366-396).
struct SrcView {
  const void* base;      // nullptr: no view (re-score from x64 or from the fp32 rows)
  int dtype;             // uml_dtype of the elements
  long long row_stride;  // in elements
  long long col_stride;  // in elements
};

#ifdef __CUDACC__
// one element of the caller's raw source chunk as float64 (exact for every dtype the ABI takes)
__device__ __forceinline__ double load_src(const SrcView& v, long long row, int f) {
  const long long i = row * v.row_stride + static_cast<long long>(f) * v.col_stride;
  switch (v.dtype) {
    case UML_F64: return static_cast<const double*>(v.base)[i];
    case UML_I64: return static_cast<double>(static_cast<const long long*>(v.base)[i]);
    case UML_I32: return static_cast<double>(static_cast<const int*>(v.base)[i]);
    case UML_U8: return static_cast<double>(static_cast<const unsigned char*>(v.base)[i]);
    default: return static_cast<double>(static_cast<const float*>(v.base)[i]);
  }
}
#endif

// Where a launch stores each row's label (device side: label_store.cuh): the local int32 vector (or nullptr), and the
// fused all-gather epilogue's peer vectors, row r of the launch at peers[i] + row_offset + r for i < n_peers
struct LabelTargets {
  int32_t* labels;
  void* peers[8];
  int n_peers;
  int wire_u8;  // 1: peer vectors are uint8 (one byte per label), 0: int32
  long long row_offset;
};

struct LinearLaunch {
  const float* x;       // device fp32 row-major
  const double* x64;    // optional fp64 copy of the same rows (lossy staging), else nullptr
  SrcView src;          // optional raw source view of the same rows (predict_host), wins over x64
  int64_t ld;           // floats per row
  int64_t ld64;
  int64_t n_rows;
  LabelTargets targets;
};

// launch `kern<<<grid, block, smem, stream>>>(p)` as a programmatic dependent of the previous kernel on the stream: its
// blocks may become resident while that kernel drains (the kernel itself waits with griddepcontrol.wait), which hides
// the launch latency between a scoring kernel and its fp64 re-score.  UML_B200_NO_PDL=1 falls back to a plain launch.
template <typename Params>
inline cudaError_t launch_dependent(void (*kern)(Params), int grid, int block, size_t smem, cudaStream_t stream, const Params& p) {
  static const bool no_pdl = getenv("UML_B200_NO_PDL") != nullptr;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(grid));
  cfg.blockDim = dim3(static_cast<unsigned>(block));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kern, p);
}

// scoring kernels (linear_kernels.cu)
// *rescore_kernel_needed: exact mode with the inline re-score switched off -> the caller launches launch_rescore_f64
// xmap: the rows as a 2-D map {F, n_rows} with {kChunkF, linear_box_rows(m.f_pad)} boxes, SWIZZLE_128B.
// half_map (optional): the batch's compact fp16 copy of the same rows, {kHalfBoxF, kTileRows} boxes, SWIZZLE_128B;
// when given and linear_half_rows_ok(m.f_pad), the kernel reads it instead of xmap (same labels, half the bytes).
// byte_map (optional, with half_map): the batch's byte copy, {kByteRowBytes, kHalfTileRows} boxes, no swizzle; the
// tensor-core schedule reads it instead of half_map.  *x_elem_bytes: the bytes per feature of the values the kernel
// multiplies (uml_stats.x_elem_bytes: 2 on either copy, 4); *x_read_bytes: the bytes per feature it reads (1, 2, 4).
cudaError_t launch_linear_tma(const CUtensorMap& xmap, const CUtensorMap* half_map, const CUtensorMap* byte_map,
                              const LinearDeviceModel& m, const LinearLaunch& l, bool exact, const FlagList& flags,
                              int sm_count, cudaStream_t stream, std::string* err, bool* rescore_kernel_needed,
                              bool half_nonneg, int* x_elem_bytes, int* x_read_bytes);
bool linear_tma_supported(const LinearDeviceModel& m, std::string* why);
// the tensor-core schedules' B operand image (LinearDeviceModel::tc_ops) and certification factor kappa of a model with
// fp64 weights w [C][F] and biases b, and its fp32 operands wt / bias; false when the model does not take them
bool build_tc_operands(const std::vector<double>& w, const std::vector<double>& b, const std::vector<float>& wt,
                       const std::vector<float>& bias, int C, int F, int f_pad, int cp, double fold_rel,
                       std::vector<uint8_t>* image, float* kappa);
cudaError_t launch_rescore_f64(const LinearDeviceModel& m, const LinearLaunch& l, const FlagList& flags, bool all_rows,
                               int sm_count, cudaStream_t stream);
// small-batch kernel of the online path (/predict, B <= 64): warp per row, fp64 straight from the raw source view
struct SmallResult {  // one per row, written by the kernel, copied back in one piece
  int32_t label;
  int32_t status;  // bit 0: NaN/Inf in the row, bit 1: fp64 margin inside the fp64 rounding bound (true tie)
};
cudaError_t launch_linear_small(const LinearDeviceModel& m, const SrcView& src, int n_rows, SmallResult* out,
                                cudaStream_t stream);
// class probabilities (LogisticRegression.predict_proba, sklearn/linear_model/_logistic.py): softmax of the scores
// (sigmoid for the binary layout), fp32 scores and exp; proba[n_rows][n_classes] row-major fp32
cudaError_t launch_linear_proba(const LinearDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, float* proba,
                                int sm_count, cudaStream_t stream);
// float64 decision_function scores (LinearClassifierMixin.decision_function, sklearn/linear_model/_base.py:366-396) of
// every row of `src` (linear_scores.cu): out[n_rows][linear_scores_width(m)] row-major, one sequential fp64 FMA chain
// per class plus the bias (DESIGN.md 3.7); rows with NaN / Inf features are counted into *nonfinite.  kind: the scores,
// or scikit-learn's float64 predict_proba / predict_log_proba of them (DESIGN.md 3.9), out[n_rows][linear_f64_width]
enum F64Output { kF64Scores = 0, kF64Proba = 1, kF64LogProba = 2 };
inline int linear_scores_width(const LinearDeviceModel& m) { return m.binary ? 1 : m.n_classes; }
inline int linear_f64_width(const LinearDeviceModel& m, int kind) {
  return kind == kF64Scores ? linear_scores_width(m) : m.n_classes;  // (n_classes is 2 for the binary layout)
}
cudaError_t launch_linear_scores_f64(const LinearDeviceModel& m, const SrcView& src, int64_t n_rows, double* out,
                                     unsigned long long* nonfinite, int sm_count, cudaStream_t stream,
                                     int kind = kF64Scores);

// 2-layer MLP (mlp_kernels.cu, mlp_tc_kernels.cu)
struct MlpHostModel {  // the caller's fp32 weights, torch nn.Linear layout
  std::vector<float> w1, b1, w2, b2;  // w1 [H][F], b1 [H], w2 [C][H], b2 [C]
};
struct MlpDeviceModel {
  const float* w1t;  // [f_pad][H + 4], column H = max_n |w1_nf|
  const float* b1;   // [H + 4], entry H = max_n |b1_n|
  const float* w2t;  // [H][cp], column C = max_c |w2_cn|
  const float* b2;   // [cp], entry C = max_c |b2_c|
  const double* rs_pack;  // fp64 operands of the re-score as one shared-memory image (mlp_rescore.cuh: mlp_rs_build_pack)
  int n_in, n_hidden, n_classes;
  int cp, f_pad;
  double w2_abs_row_sum_max;  // max_c sum_n |w2_cn|
  // tensor-core kernel: W1 split into tf32 hi | lo rows, pre-swizzled per 32-feature chunk (nullptr: not built)
  const float* w1_tiles;
  const MlpHostModel* host;
};
struct MlpTcLaunch {
  LabelTargets targets;
  long long n_rows;
  float* proba;  // launch_mlp_tc_proba: class probabilities [n_rows][n_classes] (device)
  // launch_mlp_tc_topk: [n_rows][topk_k] class indices and probabilities (device; topk_proba may be nullptr)
  int32_t* topk_idx;
  float* topk_proba;
  int topk_k;
};
// proba: the tile kernel's probability form (n_rows x n_classes fp32 instead of labels; exact and flags unused);
// topk: its top-k form (mlp_topk.cuh)
bool mlp_tma_supported(const MlpDeviceModel& m, std::string* why, bool proba = false, bool topk = false);
cudaError_t launch_mlp_tma(const CUtensorMap& xmap, const MlpDeviceModel& m, const float* x, int64_t n_rows,
                           int32_t* labels, bool exact, const FlagList& flags, int sm_count, cudaStream_t stream,
                           float* proba = nullptr);
cudaError_t launch_mlp_rescore_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows,
                                   const MlpTcLaunch& out, const FlagList& flags, bool all_rows, int sm_count,
                                   cudaStream_t stream);
bool mlp_tc_supported(const MlpDeviceModel& m, std::string* why, bool topk = false);
std::vector<float> mlp_tc_build_w1_tiles(const float* w1, int H, int F, int f_pad);
// exact: flagged rows go to the flag list; the caller launches launch_mlp_rescore_f64 behind it
cudaError_t launch_mlp_tc(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l, bool exact,
                          const FlagList& flags, int sm_count, cudaStream_t stream);
// class probabilities softmax(logits) of every row into l.proba: tensor-core kernel (rows that are tf32 values), and
// the fp64 scorer with a float64 softmax for shapes no tile kernel takes (all_rows).  Given a flag list, the
// tensor-core kernel puts the rows that are not tf32 values on it, and launch_mlp_proba_f64 without all_rows behind it
// overwrites their probabilities with the float64 route's.  No flag list: the caller knows every row is a tf32 value.
cudaError_t launch_mlp_tc_proba(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l,
                                const FlagList& flags, int sm_count, cudaStream_t stream);
cudaError_t launch_mlp_proba_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, float* proba,
                                 const FlagList& flags, bool all_rows, int sm_count, cudaStream_t stream);
// top-k class indices [n_rows][k] (and probabilities, proba != nullptr) of every row, 1 <= k <= min(C, kMlpTopkMax):
// the tile kernels' top-k forms.  exact: rows the rank guard cannot certify go to the flag list; the caller launches
// launch_mlp_topk_f64 (all_rows = false) behind them.  The tensor-core form in FAST mode, given a flag list, puts the
// rows that are not tf32 values on it (no flag list: the caller knows there are none).  launch_mlp_topk_f64 with all_rows: any shape and any k <= C.
cudaError_t launch_mlp_tc_topk(const CUtensorMap& xmap, const MlpDeviceModel& m, const MlpTcLaunch& l, bool exact,
                               const FlagList& flags, int sm_count, cudaStream_t stream);
cudaError_t launch_mlp_tma_topk(const CUtensorMap& xmap, const MlpDeviceModel& m, int64_t n_rows, int k, int32_t* idx,
                                float* proba, bool exact, const FlagList& flags, int sm_count, cudaStream_t stream);
cudaError_t launch_mlp_topk_f64(const MlpDeviceModel& m, const float* x, int64_t ld, int64_t n_rows, int k, int32_t* idx,
                                float* proba, const FlagList& flags, bool all_rows, int sm_count, cudaStream_t stream);
// top-k hits (stage_kernels.cu): first_hits[j] += rows whose target is classes[idx[row][j]] and no earlier rank's
// class; the running sum over j is the number of rows with the target among their first j + 1 classes
cudaError_t launch_topk_first_hits(const int32_t* idx, int k, int64_t n, const double* classes, int n_classes,
                                   const double* targets, unsigned long long* first_hits, cudaStream_t stream);
// small-batch kernel of the online path (B <= 64): four rows per warp through the fp64 scorer, the features read
// straight from the raw source view and cast to fp32 as the staging kernels cast them.  mlp_small_smem_bytes: its
// dynamic shared memory for the model's shape, 0 when that exceeds one SM; mlp_small_reserve sets the kernel's
// shared-memory limit (call it before a launch is captured into a graph).  kind: kSmallLabels writes out[].label;
// kSmallProba / kSmallTopk also write one record per row to rec (C fp32 probabilities, or k int32 class indices then
// their k fp32 probabilities), from the float64 softmax and ranks of mlp_topk_f64_kernel, and need the larger shared
// memory of records = true.  Every kind writes out[].status; top-k sets its bit 1 by the rank rule of that kernel.
enum SmallOutput { kSmallLabels = 0, kSmallProba = 1, kSmallTopk = 2 };
size_t mlp_small_smem_bytes(int n_in, int n_hidden, int n_classes, bool records = false);
cudaError_t mlp_small_reserve(size_t smem, bool records = false);
cudaError_t launch_mlp_small(const MlpDeviceModel& m, const SrcView& src, int n_rows, SmallResult* out, size_t smem,
                             cudaStream_t stream, int kind = kSmallLabels, int k = 0, void* rec = nullptr);
// int32 labels (device) -> every target vector of a fused exchange (int32 or uint8 wire), for kernels without peer stores
cudaError_t launch_labels_scatter(const int32_t* labels, int64_t n, const LabelTargets& out, int sm_count,
                                  cudaStream_t stream);

// staging kernels (stage_kernels.cu)
struct StageResult {  // device-side counters
  unsigned long long nonfinite;
  unsigned long long lossy;
  unsigned long long not_tf32;  // fp32 values with any of the low 13 mantissa bits set (tensor-core path needs none)
  unsigned long long not_f16;   // fp32 values that are not finite fp16 values (the compact fp16 copy needs none)
  unsigned long long negative;  // values < 0 in the compact fp16 copy (written by launch_pack_half; -0 is not one)
  unsigned long long not_u8;    // values that are not integers in [0, 255] (launch_pack_half; -0 is one, NaN is not)
};
cudaError_t launch_stage_convert(const void* src, int src_dtype, bool feature_major, int64_t src_pitch_elems,
                                 int64_t rows, int n_features, float* dst, int64_t ld, double* dst64, int64_t ld64,
                                 StageResult* result, bool check_finite, cudaStream_t stream);
// fp32 rows [rows][ld] -> fp16 rows [rows][ldh] (ldh = linear_half_ld(F), columns >= F zero); exact when the staging
// pass found not_f16 == 0
// (*negative is raised when any value is < 0: the tensor-core schedule needs none; *not_u8 when any value is not an
// integer in [0, 255]: the byte copy needs none)
cudaError_t launch_pack_half(const float* x, int64_t ld, int64_t rows, int n_features, void* xh, int64_t ldh,
                             unsigned long long* negative, unsigned long long* not_u8, cudaStream_t stream);
// fp32 rows [rows][ld] -> byte rows [rows][kByteRowBytes], feature f at byte linear_byte_pos(f), zeros past F; exact
// when launch_pack_half found not_u8 == 0 (-0 becomes byte 0)
cudaError_t launch_pack_bytes(const float* x, int64_t ld, int64_t rows, int n_features, void* xb, cudaStream_t stream);

}  // namespace uml
