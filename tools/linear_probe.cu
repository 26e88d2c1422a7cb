// Where the time of the linear tile kernel goes, on 10M x 64 fp32 rows (2.56 GB, the cfg2 shape), on their compact
// fp16 copy (1.28 GB) and on their byte copy (0.64 GB), against the card's own read ceiling.  Built eleven times by
// tools/linear_probe.sh from linear_kernels.cu itself:
//   plain                   read ceiling (streaming 16-byte non-allocating loads) over 2.56 GB, 1.28 GB and 0.64 GB +
//                           the tile kernel, the three CUDA-core schedules and both tensor-core ones (kHalfMma on the
//                           fp16 rows, kByteMma on the byte rows; B operand and kappa from build_tc_operands)
//   -DUML_PROBE_FEED_ONLY   the same producer, ring, order and barriers with consumers that skip the math, under
//                           L2_PROMOTION_256B (what the library encodes) and L2_PROMOTION_NONE; also the byte
//                           schedule's ring of 16 KiB {64 bytes, 256 rows} stages
//   -DUML_PROBE_WAIT_CLOCKS the tile kernel with clock64() totals around the producer's `empty` and the scoring
//                           warps' `full` waits, over the time the scoring warps hold a landed stage, and over the time
//                           the re-score warp spends on rows from the queue (its busy fraction, split into the fp32
//                           replay and the fp64 re-score), and the rows tier 1 queued per launch; every schedule
//   -DUML_PROBE_TIMELINE    the tile kernel with %globaltimer stamps per CTA (entry, first issue, first landing, last
//                           release, exit; in the tensor-core schedules also the first drain warp to see every
//                           publisher done, the last batch claimed, the last replay and the last fp64 row finished) over
//                           two back-to-back launches: ramp, exit spread, launch gap, and where the tail goes
//   -DUML_PROBE_NO_W, -DUML_PROBE_NO_X, both   the fp16 schedule without its W loads, without its x loads and
//                           conversions, and with neither (the FMAs and the epilogue alone): which of the scoring
//                           warps' operands the time above the feed pays for.  Wrong scores by design.
//   -DUML_PROBE_NO_EPILOGUE, -DUML_PROBE_NO_HANDOFF   the byte schedule alone, without its per-item epilogue (wgmma
//                           and stage release only) and with tier 1's verdict forced to "certified" (no queue hand-off)
//   -DUML_PROBE_HALF_ONLY   the fp16 schedule alone, and once more with -DUML_PROBE_HALF_PASS_ROWS=4 (256-row stages
//                           scored in two passes of 4 rows per lane by the same four warps): the script runs the two
//                           alternately, which separates the W reuse of 8 rows per lane from the warp count
// Every figure is CUDA-event time over >= 0.5 s of back-to-back launches.  Prints one JSON object per line.
#include "../unionml_b200/csrc/linear_kernels.cu"

#include <cudaTypedefs.h>

#include <cmath>
#include <vector>

using namespace uml;

#define CK(x)                                                                               \
  do {                                                                                      \
    cudaError_t e_ = (x);                                                                   \
    if (e_ != cudaSuccess) {                                                                \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));    \
      exit(1);                                                                              \
    }                                                                                       \
  } while (0)

static const long long kRows = 10000000;
static const int kF = 64, kC = 10;

__global__ void fill_kernel(float* x, __half* xh, uint8_t* xb, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned h = static_cast<unsigned>(i) * 2654435761u;
    h ^= h >> 15;
    x[i] = static_cast<float>(h % 17u);  // digits-like pixel values 0..16
    xh[i] = __float2half_rn(x[i]);       // the same values, exactly (what the engine's pack kernel writes)
    xb[i / kF * kByteRowBytes + linear_byte_pos(static_cast<int>(i % kF))] = static_cast<uint8_t>(h % 17u);
  }
}

// streaming read: 16-byte non-allocating loads, four in flight per thread, folded into one word per thread so no
// load can be dropped; the block's clock64() span over its lifetime gives the SM clock under this load
__global__ void __launch_bounds__(512) read_kernel(const uint4* __restrict__ x, long long n16, unsigned* sink,
                                                   long long* cycles) {
  const long long t0 = clock64();
  unsigned acc = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v[k].x), "=r"(v[k].y), "=r"(v[k].z), "=r"(v[k].w)
                   : "l"(x + i + k * stride));
#pragma unroll
    for (int k = 0; k < 4; ++k) acc ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
  }
  for (; i < n16; i += stride) {
    const uint4 v = x[i];
    acc ^= v.x ^ v.y ^ v.z ^ v.w;
  }
  if (acc == 0x9e3779b9u) sink[0] = acc;
  if (blockIdx.x == 0 && threadIdx.x == 0) *cycles = clock64() - t0;
}

static PFN_cuTensorMapEncodeTiled_v12000 encoder() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
}

// fp32 rows: {32, box_rows} boxes; fp16 rows (elem 2): {64, 128} boxes; byte rows (elem 1): {64, 256} boxes without
// swizzle, as the engine encodes them
static CUtensorMap make_map(const void* x, int box_rows, CUtensorMapL2promotion promo, int elem = 4) {
  CUtensorMap map{};
  cuuint64_t gdim[2] = {(cuuint64_t)kF, (cuuint64_t)kRows};
  cuuint64_t gstride[1] = {(cuuint64_t)kF * elem};
  cuuint32_t box[2] = {(cuuint32_t)(elem == 4 ? kChunkF : kHalfBoxF), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encoder()(&map, elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : elem == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                                                                     : CU_TENSOR_MAP_DATA_TYPE_UINT8,
                         2, (void*)x, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         elem == 1 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, promo,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "cuTensorMapEncodeTiled: %d\n", (int)r);
    exit(1);
  }
  return map;
}

// mean ms per launch of fn() over >= 0.5 s (after a warm-up launch sized the count)
template <typename FN>
static double time_ms(FN fn) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) fn();
  CK(cudaEventRecord(a));
  fn();
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float one = 0.f;
  CK(cudaEventElapsedTime(&one, a, b));
  const int n = std::max(100, static_cast<int>(std::ceil(600.0 / std::max(one, 0.01f))));
  CK(cudaEventRecord(a));
  for (int i = 0; i < n; ++i) fn();
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, a, b));
  CK(cudaGetLastError());
  return ms / n;
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const double bytes = static_cast<double>(kRows) * kF * 4;
  float* x = nullptr;
  __half* xh = nullptr;
  uint8_t* xb = nullptr;
  CK(cudaMalloc(&x, static_cast<size_t>(bytes)));
  CK(cudaMalloc(&xh, static_cast<size_t>(bytes / 2)));
  CK(cudaMalloc(&xb, static_cast<size_t>(bytes / 4)));
  fill_kernel<<<prop.multiProcessorCount * 8, 512>>>(x, xh, xb, kRows * kF);
  CK(cudaDeviceSynchronize());

#if defined(UML_PROBE_NO_W) || defined(UML_PROBE_NO_X)
#define UML_PROBE_HALF_ONLY
#endif
#if defined(UML_PROBE_NO_W) && defined(UML_PROBE_NO_X)
  const char* build = "math_only";
#elif defined(UML_PROBE_NO_W)
  const char* build = "no_w_loads";
#elif defined(UML_PROBE_NO_X)
  const char* build = "no_x_loads";
#elif defined(UML_PROBE_NO_EPILOGUE)
  const char* build = "no_epilogue";
#elif defined(UML_PROBE_NO_HANDOFF)
  const char* build = "no_handoff";
#elif defined(UML_PROBE_FEED_ONLY)
  const char* build = "feed_only";
#elif defined(UML_PROBE_WAIT_CLOCKS)
  const char* build = "wait_clocks";
#elif defined(UML_PROBE_TIMELINE)
  const char* build = "timeline";
#elif defined(UML_PROBE_HALF_ONLY) && defined(UML_PROBE_HALF_PASS_ROWS)
  const char* build = "half_only_rows4";
#elif defined(UML_PROBE_HALF_ONLY)
  const char* build = "half_only";
#else
  const char* build = "plain";
  {
    unsigned* sink = nullptr;
    long long* cyc = nullptr;
    CK(cudaMalloc(&sink, 4));
    CK(cudaMalloc(&cyc, 8));
    const int grid = prop.multiProcessorCount * 4;  // 2048 threads per SM resident, 64 KB of loads in flight per SM
    // the byte copy's 0.64 GB and the fp16 copy's 1.28 GB first, then the fp32 rows' 2.56 GB: the last read_ceiling
    // line is what MEASURED_PEAKS.json records
    for (const double part : {0.25, 0.5, 1.0}) {
      const double b = bytes * part;
      const double ms = time_ms([&] {
        read_kernel<<<grid, 512>>>(reinterpret_cast<const uint4*>(x), static_cast<long long>(b) / 16, sink, cyc);
      });
      long long cycles = 0;
      CK(cudaMemcpy(&cycles, cyc, 8, cudaMemcpyDeviceToHost));
      printf("{\"probe\": \"read_ceiling\", \"device\": \"%s\", \"bytes\": %.0f, \"ms\": %.4f, \"hbm_gbs\": %.1f, "
             "\"sm_clock_mhz_under_load\": %.0f}\n",
             prop.name, b, ms, b / ms * 1e-6, cycles / (ms * 1e3));
    }
  }
#endif

  // the cfg2 model shape: 10 classes, wt [64][cp] with the wmax column, bias [cp] with max|b|
  const int cp = (kC + 1 + 3) / 4 * 4;
  std::vector<float> wt(static_cast<size_t>(kF) * cp, 0.f), bias(cp, 0.f);
  // b64 holds 2C doubles as in upload_model: the biases, then the bias magnitudes score_row_f64's bound reads
  std::vector<double> w64(static_cast<size_t>(kF) * linear_w64_stride(kC), 0.0), b64(2 * kC, 0.0);
  unsigned s = 12345u;
  auto rnd = [&] {
    s = s * 1664525u + 1013904223u;
    return (static_cast<float>(s >> 8) / 16777216.f - 0.5f) * 0.1f;
  };
  for (int f = 0; f < kF; ++f) {
    float wmax = 0.f;
    for (int c = 0; c < kC; ++c) {
      const float v = rnd();
      wt[f * cp + c] = v;
      w64[static_cast<size_t>(f) * linear_w64_stride(kC) + c] = v;
      wmax = fmaxf(wmax, fabsf(v));
    }
    wt[f * cp + kC] = wmax;
  }
  float bmax = 0.f;
  for (int c = 0; c < kC; ++c) {
    bias[c] = rnd() * 10.f;
    b64[c] = bias[c];
    b64[kC + c] = fabs(static_cast<double>(bias[c]));
    bmax = fmaxf(bmax, fabsf(bias[c]));
  }
  bias[kC] = bmax;
  LinearDeviceModel m{};
  float *d_wt, *d_bias;
  double *d_w64, *d_b64;
  CK(cudaMalloc(&d_wt, wt.size() * 4));
  CK(cudaMalloc(&d_bias, bias.size() * 4));
  CK(cudaMalloc(&d_w64, w64.size() * 8));
  CK(cudaMalloc(&d_b64, b64.size() * 8));
  CK(cudaMemcpy(d_wt, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_bias, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_w64, w64.data(), w64.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_b64, b64.data(), b64.size() * 8, cudaMemcpyHostToDevice));
  m.wt = d_wt;
  m.bias = d_bias;
  m.w64 = d_w64;
  m.b64 = d_b64;
  m.w64_stride = linear_w64_stride(kC);
  m.n_classes = kC;
  m.n_features = kF;
  m.cp = cp;
  m.f_pad = kF;
  uint8_t* labels = nullptr;
  unsigned long long* counters = nullptr;
  CK(cudaMalloc(&labels, kRows));
  CK(cudaMalloc(&counters, 24 * sizeof(unsigned long long)));  // the kernel's slots, then probe_clocks from 8
  CK(cudaMemset(counters, 0, 24 * sizeof(unsigned long long)));
#ifdef UML_PROBE_TIMELINE
  unsigned long long* timeline = nullptr;  // [2 launches][grid][kProbeStamps]
  const size_t timeline_words = 2 * static_cast<size_t>(prop.multiProcessorCount) * kProbeStamps;
  CK(cudaMalloc(&timeline, timeline_words * sizeof(unsigned long long)));
  // stamp 5 is a minimum over the drain warps, the others are stores or maxima
  std::vector<unsigned long long> timeline_init(timeline_words, 0ull);
  for (size_t i = 5; i < timeline_words; i += kProbeStamps) timeline_init[i] = ~0ull;
  auto reset_timeline = [&] {
    CK(cudaMemcpy(timeline, timeline_init.data(), timeline_words * sizeof(unsigned long long), cudaMemcpyHostToDevice));
  };
  reset_timeline();
#endif

  // the EXACT + QUEUE kernel bench.py runs (uint8 labels to one target), in each schedule
  // the tensor-core schedules' B operand and kappa, as the engine builds them at model load
  std::vector<double> w_cf(static_cast<size_t>(kC) * kF), b_c(kC);
  for (int c = 0; c < kC; ++c) {
    b_c[c] = bias[c];
    for (int f = 0; f < kF; ++f) w_cf[static_cast<size_t>(c) * kF + f] = wt[f * cp + c];
  }
  std::vector<uint8_t> tc_image;
  float tc_kappa = 0.f;
  if (!build_tc_operands(w_cf, b_c, wt, bias, kC, kF, kF, cp, 0.0, &tc_image, &tc_kappa)) {
    fprintf(stderr, "build_tc_operands refused the probe's model\n");
    exit(1);
  }
  void* d_tc = nullptr;
  CK(cudaMalloc(&d_tc, tc_image.size()));
  CK(cudaMemcpy(d_tc, tc_image.data(), tc_image.size(), cudaMemcpyHostToDevice));
  auto run = [&](LinearSched sched, CUtensorMapL2promotion promo, const char* promo_name) {
    const bool whole = sched == LinearSched::kWhole, half = sched == LinearSched::kHalf;
    const bool byte = sched == LinearSched::kByteMma, tc = linear_tc_sched(sched);
    const bool f16 = half || sched == LinearSched::kHalfMma;
    const int tile = whole ? kWholeTileRows : f16 || byte ? kHalfTileRows : kTileRows;
    const CUtensorMap map = byte ? make_map(xb, kHalfTileRows, promo, 1)
                            : f16 ? make_map(xh, kTileRows, promo, 2) : make_map(x, tile, promo);
    const double read_bytes = byte ? bytes / 4 : f16 ? bytes / 2 : bytes;
    TmaKernelParams p{};
    p.wt = m.wt;
    p.bias = m.bias;
    p.targets.peers[0] = labels;
    p.targets.n_peers = 1;
    p.targets.wire_u8 = 1;
    p.n_rows = kRows;
    p.num_tiles = (kRows + tile - 1) / tile;
    p.f_pad = kF;
    p.kc = kF / kChunkF;
    const size_t fixed = tma_fixed_smem(m, f16 || byte) + (tc ? linear_tc_b_bytes(kC) : 0) + linear_epi_bytes(sched, kC);
    const int stage_bytes = linear_stage_bytes(sched);
    p.num_stages = std::min(64, static_cast<int>((kMaxSmemBytes - fixed) / stage_bytes));
    p.thr = static_cast<float>(2.0 * (kF + 4.0) * 5.9604644775390625e-08 * (1.0 + kF * 4.76837158203125e-07) * 1.0001);
    p.x = x;
    p.ld = kF;
    p.w64 = m.w64;
    p.w64_stride = m.w64_stride;
    p.b64 = m.b64;
    p.n_classes = kC;
    p.n_features = kF;
    p.fold_rel = m.fold_rel;  // 0: no affine fold
    p.binary = m.binary;      // 0: ten classes
    p.counters = counters;
    p.tc_ops = d_tc;
    p.tc_kappa = tc_kappa;
#ifdef UML_PROBE_WAIT_CLOCKS
    p.probe_clocks = counters + 8;
#endif
#ifdef UML_PROBE_TIMELINE
    p.probe_timeline = timeline;
#endif
    const size_t smem = fixed + static_cast<size_t>(p.num_stages) * stage_bytes;
    const int grid = prop.multiProcessorCount;
    auto launch = [&] {
      const cudaError_t err = byte    ? launch_one<kC, true, true, LinearSched::kByteMma>(map, p, grid, smem, 0)
                              : tc    ? launch_one<kC, true, true, LinearSched::kHalfMma>(map, p, grid, smem, 0)
                              : half  ? launch_one<kC, true, true, LinearSched::kHalf>(map, p, grid, smem, 0)
                              : whole ? launch_one<kC, true, true, LinearSched::kWhole>(map, p, grid, smem, 0)
                                      : launch_one<kC, true, true, LinearSched::kChunked>(map, p, grid, smem, 0);
      CK(err);
    };
    const double ms = time_ms(launch);
    printf("{\"probe\": \"tile_kernel\", \"build\": \"%s\", \"schedule\": \"%s\", \"l2_promotion\": \"%s\", \"stages\": %d, "
           "\"scoring_warps\": %d, \"rows_per_lane_per_pass\": %d, \"ms\": %.4f, \"bytes_read\": %.0f, \"gbs\": %.1f",
           build, byte ? "byte_rows_tc_256x64" : tc ? "half_rows_tc_256x64" : half ? "half_rows_256x64"
                  : whole ? "whole_rows_64" : "chunked_128x32",
           promo_name, p.num_stages, linear_consumer_warps(sched), half ? kHalfPassRows : tile / 32, ms, read_bytes,
           read_bytes / ms * 1e-6);
#ifdef UML_PROBE_WAIT_CLOCKS
    // one more launch with the totals cleared: fractions of the producer's / scoring warps' own loop time
    CK(cudaMemset(counters + 8, 0, 12 * sizeof(unsigned long long)));
    unsigned long long flagged0 = 0, flagged1 = 0;
    CK(cudaMemcpy(&flagged0, counters + kCounterFlagged, 8, cudaMemcpyDeviceToHost));
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    CK(cudaEventRecord(a));
    launch();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float one = 0.f;
    CK(cudaEventElapsedTime(&one, a, b));
    unsigned long long c[12];
    CK(cudaMemcpy(c, counters + 8, sizeof(c), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&flagged1, counters + kCounterFlagged, 8, cudaMemcpyDeviceToHost));
    // mean stages per CTA landed and not yet released (one scoring warp per stage, four in the tensor-core
    // schedules): the scoring warps' summed hold time over one warp's loop time, per CTA
    // (kByteMma: the MMA warps; its epilogue warps report in [8] and [9])
    const int scoring_warps = grid * (tc ? 4 * linear_ring_units(sched) : linear_consumer_warps(sched));
    const double held_stages =
        static_cast<double>(c[4]) / (static_cast<double>(c[3]) / scoring_warps) / grid / (tc ? 4 : 1);
    printf(", \"producer_empty_wait_frac\": %.4f, \"consumer_full_wait_frac\": %.4f, \"held_stages\": %.3f, "
           "\"ring_stages\": %d, \"sm_clock_mhz_under_load\": %.0f, \"rescore_warp_busy_frac\": %.4f, "
           "\"rescore_warp_replay_frac\": %.4f, \"rescore_warp_fp64_frac\": %.4f, \"rows_queued_per_launch\": %llu, "
           "\"rows_fp64_per_launch\": %llu",
           static_cast<double>(c[0]) / c[1], static_cast<double>(c[2]) / c[3], held_stages,
           p.num_stages, static_cast<double>(c[1]) / grid / (one * 1e3), c[6] ? static_cast<double>(c[5]) / c[6] : 0.0,
           c[6] ? static_cast<double>(c[5] - c[10]) / c[6] : 0.0, c[6] ? static_cast<double>(c[10]) / c[6] : 0.0, c[11],
           flagged1 - flagged0);
    if (byte)  // MMA warps' waits for a free score slot over their loop; epilogue warps' waits for a full one over theirs
      printf(", \"mma_slot_wait_frac\": %.4f, \"epilogue_full_wait_frac\": %.4f", static_cast<double>(c[7]) / c[3],
             c[9] ? static_cast<double>(c[8]) / c[9] : 0.0);
#endif
#ifdef UML_PROBE_TIMELINE
    // two launches back to back, each stamping its own [grid][kProbeStamps] block
    reset_timeline();
    CK(cudaDeviceSynchronize());
    launch();
    p.probe_timeline = timeline + static_cast<size_t>(grid) * kProbeStamps;
    launch();
    p.probe_timeline = timeline;
    CK(cudaDeviceSynchronize());
    std::vector<unsigned long long> t(timeline_words);
    CK(cudaMemcpy(t.data(), timeline, timeline_words * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    auto col = [&](int launch_k, int slot) {
      std::vector<double> v(grid);
      for (int b = 0; b < grid; ++b) v[b] = static_cast<double>(t[(static_cast<size_t>(launch_k) * grid + b) * kProbeStamps + slot]);
      return v;
    };
    auto median = [](std::vector<double> v) {
      std::sort(v.begin(), v.end());
      return v[v.size() / 2];
    };
    for (int k = 0; k < 2; ++k) {
      const std::vector<double> entry = col(k, 0), issue = col(k, 1), land = col(k, 2), rel = col(k, 3), ex = col(k, 4);
      std::vector<double> ramp(grid), first_issue(grid), tail(grid);
      for (int b = 0; b < grid; ++b) {
        ramp[b] = land[b] - entry[b];
        first_issue[b] = issue[b] - entry[b];
        tail[b] = ex[b] - rel[b];
      }
      const double e0 = *std::min_element(entry.begin(), entry.end());
      const double x0 = *std::min_element(ex.begin(), ex.end()), x1 = *std::max_element(ex.begin(), ex.end());
      printf(", \"launch%d\": {\"span_us\": %.2f, \"entry_spread_us\": %.2f, \"first_issue_us_median\": %.2f, "
             "\"ramp_us_median\": %.2f, \"ramp_us_max\": %.2f, \"exit_spread_us_max\": %.2f, "
             "\"exit_spread_us_median\": %.2f, \"last_release_to_exit_us_median\": %.2f, "
             "\"last_release_to_exit_us_max\": %.2f}",
             k, (x1 - e0) * 1e-3, (*std::max_element(entry.begin(), entry.end()) - e0) * 1e-3,
             median(first_issue) * 1e-3, median(ramp) * 1e-3, *std::max_element(ramp.begin(), ramp.end()) * 1e-3,
             (x1 - x0) * 1e-3, (median(ex) - x0) * 1e-3, median(tail) * 1e-3,
             *std::max_element(tail.begin(), tail.end()) * 1e-3);
      if (tc) {
        // the tail after the last release, stamp by stamp: median and maximum over the CTAs that have the stamp
        // (a CTA whose drain took no batch has no claim, replay or fp64 stamp)
        const std::vector<double> done = col(k, 5), claim = col(k, 6), replay = col(k, 7), f64 = col(k, 8);
        auto after = [&](const std::vector<double>& v, const char* key) {
          std::vector<double> d;
          for (int b = 0; b < grid; ++b)
            if (v[b] > 0.0 && v[b] < 1.8e19) d.push_back(v[b] - rel[b]);
          if (d.empty()) return;
          printf(", \"%s_us_median\": %.2f, \"%s_us_max\": %.2f, \"%s_ctas\": %zu", key, median(d) * 1e-3, key,
                 *std::max_element(d.begin(), d.end()) * 1e-3, key, d.size());
        };
        printf(", \"launch%d_tail\": {\"last_release_to_exit_us_median\": %.2f", k, median(tail) * 1e-3);
        after(done, "all_published");
        after(claim, "last_claim");
        after(replay, "last_replay_done");
        after(f64, "last_fp64_done");
        std::vector<double> work_end(grid);  // the drain's last work (replay or fp64) to exit
        std::vector<double> d;
        for (int b = 0; b < grid; ++b) {
          const double w = std::max(replay[b], f64[b]);
          if (w > 0.0) d.push_back(ex[b] - w);
        }
        if (!d.empty())
          printf(", \"drain_end_to_exit_us_median\": %.2f, \"drain_end_to_exit_us_max\": %.2f", median(d) * 1e-3,
                 *std::max_element(d.begin(), d.end()) * 1e-3);
        printf("}");
      }
    }
    {
      const std::vector<double> ex0 = col(0, 4), entry1 = col(1, 0);
      std::vector<double> all;
      for (int k = 0; k < 2; ++k)
        for (int s = 0; s < 5; ++s)  // (the drain stamps are absent in the CUDA-core schedules)
          for (double v : col(k, s)) all.push_back(v);
      std::sort(all.begin(), all.end());
      double quantum = 0.0;  // the smallest step between distinct stamps: the timer's resolution, or finer
      for (size_t i = 1; i < all.size(); ++i)
        if (all[i] > all[i - 1] && (quantum == 0.0 || all[i] - all[i - 1] < quantum)) quantum = all[i] - all[i - 1];
      printf(", \"launch_gap_us\": %.2f, \"timer_step_ns_min\": %.0f",
             (*std::min_element(entry1.begin(), entry1.end()) - *std::max_element(ex0.begin(), ex0.end())) * 1e-3,
             quantum);
    }
#endif
    printf("}\n");
    fflush(stdout);
  };
#ifdef UML_PROBE_HALF_ONLY
  run(LinearSched::kHalf, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  return 0;
#endif
#if defined(UML_PROBE_NO_EPILOGUE) || defined(UML_PROBE_NO_HANDOFF)
  run(LinearSched::kByteMma, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  return 0;
#endif
  run(LinearSched::kChunked, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  run(LinearSched::kWhole, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  run(LinearSched::kHalf, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  run(LinearSched::kHalfMma, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
  run(LinearSched::kByteMma, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "256B");
#ifdef UML_PROBE_FEED_ONLY
  run(LinearSched::kChunked, CU_TENSOR_MAP_L2_PROMOTION_NONE, "none");
  run(LinearSched::kWhole, CU_TENSOR_MAP_L2_PROMOTION_NONE, "none");
  run(LinearSched::kHalf, CU_TENSOR_MAP_L2_PROMOTION_NONE, "none");
#endif
  return 0;
}
