// ground.cu -- slope-based polar-grid ground removal on sm_90a.
//
// Replaces groundRemove (/root/reference/object_tracking/src/groundremove/ground_removal.cpp:177-249) and
// gaussSmoothen (src/groundremove/gaus_blur.cpp:52-68) with ONE cooperative kernel per frame, ground_fused_kernel:
//
//   phase 1  every CTA owns a contiguous chunk of the XYZI frame and pulls it into shared memory with the bulk async
//            copy engine (TMA, one cp.async.bulk per 16 KB tile); range filter (:46-64), bit-exact point->cell
//            (:67-76, exact_math.cuh), warp-aggregated atomicMin of an order-preserving key into the 80x120
//            min-z grid (:79-92).  The points and their u16 cell ids STAY in shared memory.
//   -- grid barrier --
//   phase 2  the 80 channels are split over the first min(G,80) CTAs (one halo channel per side recomputed locally):
//            height clamp (:192-197), 3-tap blur in fp64 (gaus_blur.cpp), hDiff (:95-117), ground flag (:205-214),
//            median filter (:120-146, Jacobi -- provably order independent), outlier filter (:149-174, closed form).
//   -- grid barrier --
//   phase 3  ground / elevated decision (:221-247) from shared memory + ORDER-PRESERVING compaction of both output
//            clouds (per-CTA totals published once, every CTA sums its predecessors), fused with the first pass of
//            clustering (cartesian cell + occupancy of every elevated point, component_clustering.cpp:38-47).
//
// HBM traffic is the compulsory minimum: every input point is read once (16 B) and every surviving point written
// once (16 B); the reference, and a kernel-per-stage design, read the frame twice and round-trip the cell ids.
//
// Everything that decides a cell index or a label is IEEE round-to-nearest without FMA contraction, so the
// results are bit-identical to the reference built for x86-64.
#include <climits>
#include <cstring>
#include <mutex>
#include "lmot_internal.cuh"
#include "exact_math.cuh"
#include "tma.cuh"
#include "ccl_device.cuh"
#include "ground_lines.cuh"
#include "polar_cell.cuh"

namespace lmot {

namespace {

std::mutex g_ground_mutex;                 // one ground kernel in flight per device (see ground_launch_batch)
// the chain of ground kernels of a device: every launch waits for the previous one.  On the same stream that is stream order; on
// another stream it is `done`, recorded right behind the launch -- or, for the stand-alone entry points (`chain`), only when a
// launch on another stream needs it: kernel / event record / kernel costs a launch latency more per launch than kernel / kernel.
struct GroundChain {
  cudaEvent_t done = nullptr;
  cudaStream_t last = nullptr;
  bool have_last = false, recorded = false, record_pending = false;
};
GroundChain g_chain[64];

__device__ __forceinline__ unsigned fkey(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// The cell index must equal the exact evaluation above bit for bit, but ~170 instructions per point (two IEEE divisions,
// an IEEE square root, an 11-term polynomial without FMA, an fp64 divide) make the kernel instruction-bound.  The exact
// path is only needed where it can matter.  Fast path: d ~ d2 * rsqrt(d2) (MUFU, <= 2 ulp), the scaled bin coordinate
// t = (d - rMin) * 120/(rMax - rMin), the angle from a degree-6 minimax polynomial of atan on [0,1] with octant folding
// (|error| < 6e-7 rad), scaled to channel units.  Measured against the exact evaluation over 2e7 points (random, tiny
// and huge |y/x|): the fast coordinates differ from the reference's by < 1.6e-5 channel widths and < 6.2e-5 bin
// widths.  A point whose fast coordinates lie further than kChanGuard = 2e-4 / kBinGuard = 6e-4 (>= 10x those bounds)
// from every integer has the same floor() under both evaluations, and the range filter `rMin < d < rMax` is the same
// statement as 0 < t < 120; every other point (about 1.6 in 1000; NaN/Inf/zero-radius inputs fail the comparisons and
// land there too) is re-evaluated exactly.  tests/test_ground_gpu.py compares cells of random, HDL-64 and
// boundary-hugging clouds (down to 1e-7 rad / 1e-6 m from the boundaries) against the reference bit for bit.
constexpr float kChanGuard = 2.0e-4f;
constexpr float kBinGuard = 6.0e-4f;

__device__ __forceinline__ uint16_t polar_cell(float x, float y, const GroundParams& p) {
  const float d2 = fadd(fmul(x, x), fmul(y, y));
  const float t = __fmaf_rn(d2, rsqrtf(d2), -p.r_min) * p.bin_scale;
  const float ax = fabsf(x), ay = fabsf(y);
  const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
  const float z = __fdividef(mn, mx);
  const float u = z * z;
  float a = 0.00782548263669014f;
  a = __fmaf_rn(a, u, -0.03689862787723541f);
  a = __fmaf_rn(a, u, 0.08374155312776566f);
  a = __fmaf_rn(a, u, -0.13480405509471893f);
  a = __fmaf_rn(a, u, 0.19879871606826782f);
  a = __fmaf_rn(a, u, -0.3332637548446655f);
  a = __fmaf_rn(a, u, 0.9999993443489075f);
  a = a * z;
  if (ay > ax) a = 1.57079632679489661923f - a;
  if (x < 0.f) a = 3.14159265358979323846f - a;
  if (y < 0.f) a = -a;
  const float sc = __fmaf_rn(a, (float)(kNumChannel / 6.28318530717958647692), (float)(kNumChannel / 2));
  if (t < -kBinGuard || t > (float)kNumBin + kBinGuard) return kNoCell;      // certainly outside (rMin, rMax)
  const float tf = floorf(t), cf = floorf(sc);
  const float tr = t - tf, cr = sc - cf;
  if (!(tr > kBinGuard && tr < 1.0f - kBinGuard && cr > kChanGuard && cr < 1.0f - kChanGuard)) return polar_cell_exact(x, y, p);
  return (uint16_t)((int)cf * kNumBin + (int)tf);
}

// generic-stride input -> float4 (the hot path is stride 4 and never runs this)
__global__ void repack_kernel(const float* __restrict__ in, int n, int stride, float4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = make_float4(in[(size_t)i * stride], in[(size_t)i * stride + 1], in[(size_t)i * stride + 2], 1.f);
}

// ---------------------------------------------------------------------------------------------------------------
// polar-grid stages for a window of channels.  H / G: shared-memory height and ground flag of the window's cells,
// window = the CTA's own channels [own0, own0 + n_own) plus one halo channel on each side (the 80 channels are
// independent in every stage except the median filter, which looks one channel to each side; the halo's clamp / blur /
// hDiff / flag stages are recomputed locally, so the CTAs never exchange grid data).
constexpr int kFusedThreads = 1024;                 // threads per CTA == points per tile
constexpr int kMinCtas = 8;                         // => at most 10 own + 2 halo channels per CTA
constexpr int kMaxLocChan = kNumChannel / kMinCtas + 2;
constexpr int kMaxLocCells = kMaxLocChan * kNumBin;  // 1440
constexpr int kCellsPerThread = (kMaxLocCells + kFusedThreads - 1) / kFusedThreads;   // 2

// ground_removal.cpp:236-246 labels a point ground iff  (double)z < (double)hGround + 0.25  and its cell is a ground cell.  The
// right-hand side depends on the cell only: this is the largest float `lim` with (double)lim < (double)h + tol, so that the
// per-point test is ONE float compare, z <= lim (identical for every float z; NaN for non-ground cells: never true).
__device__ __forceinline__ float label_limit(float h, bool is_ground, double tol) {
  if (!is_ground) return __int_as_float(0x7FC00000);
  const double thr = __dadd_rn((double)h, tol);
  float f = __double2float_rd(thr);                    // largest float <= thr
  if ((double)f == thr) {                              // ... but the test is strict: step to the next float below
    const int b = __float_as_int(f);
    f = (f == 0.f) ? __int_as_float(0x80000001) : __int_as_float(b > 0 ? b - 1 : b + 1);
  }
  return f;
}

// t_hmin / t_hmax / h_sensor: lmot_params' values, or the frame's sensor's in a rig launch (lmot_set_sensors)
__device__ __forceinline__ void polar_grid_slice(const GroundParams& p, float t_hmin, float t_hmax, float h_sensor, const unsigned* __restrict__ keys, int own0, int n_own,
                                                 float* H, uint8_t* G, float* __restrict__ o_minz, float* __restrict__ o_height,
                                                 float* __restrict__ o_smoothed, float* __restrict__ o_hdiff,
                                                 float* __restrict__ o_hg, float* __restrict__ o_lim = nullptr) {
  const int tid = threadIdx.x;
  const int ch0 = own0 - 1;                                   // global channel of local channel 0 (may be -1)
  const int n_cells = (n_own + 2) * kNumBin;

  // (a4) height clamp, ground_removal.cpp:192-197
#pragma unroll
  for (int j = 0; j < kCellsPerThread; ++j) {
    const int l = tid + j * kFusedThreads;
    if (l < n_cells) {
      const int lc = l / kNumBin, b = l - lc * kNumBin, ch = ch0 + lc;
      float h = 0.f;
      if (ch >= 0 && ch < kNumChannel) {
        const float zi = fkey_inv(__ldcg(&keys[ch * kNumBin + b]));
        if (lc >= 1 && lc <= n_own && o_minz) o_minz[ch * kNumBin + b] = zi;
        if (zi > t_hmin && zi < t_hmax) h = zi;
        else if (zi > t_hmax) h = h_sensor;
        else h = t_hmin;
      }
      H[l] = h;
    }
  }
  __syncthreads();

  // (a5) blur, (a6) hDiff, (a7) ground flag -- per channel, neighbours along bin
#pragma unroll
  for (int j = 0; j < kCellsPerThread; ++j) {
    const int l = tid + j * kFusedThreads;
    if (l < n_cells) {
      const int lc = l / kNumBin, b = l - lc * kNumBin, ch = ch0 + lc;
      uint8_t g = 0;
      if (ch >= 0 && ch < kNumChannel) {
        const float h = H[l];
        double acc = 0.0;                                       // gaus_blur.cpp:58-65, order j = i-1, i, i+1
        if (b > 0) acc = __dadd_rn(acc, __dmul_rn(p.tap[0], (double)H[l - 1]));
        acc = __dadd_rn(acc, __dmul_rn(p.tap[1], (double)h));
        if (b < kNumBin - 1) acc = __dadd_rn(acc, __dmul_rn(p.tap[2], (double)H[l + 1]));
        const float sm = (float)acc;
        float hd;                                               // ground_removal.cpp:95-117
        if (b == 0) hd = fsub(h, H[l + 1]);
        else if (b == kNumBin - 1) hd = fsub(h, H[l - 1]);
        else {
          const float pre = fsub(h, H[l - 1]), post = fsub(h, H[l + 1]);
          hd = (pre > post) ? pre : post;
        }
        if (lc >= 1 && lc <= n_own && o_smoothed) { o_smoothed[ch * kNumBin + b] = sm; o_hdiff[ch * kNumBin + b] = hd; }
        g = ((sm < t_hmax && hd < p.t_hdiff) || (h < t_hmax && hd < p.t_hdiff)) ? 1 : 0;  // :205-214
      }
      G[l] = g;
    }
  }
  __syncthreads();

  // (a8) applyMedianFilter, ground_removal.cpp:120-146.  A cell flips only if its four neighbours are ground
  // already, and a neighbour that flips in this pass would have needed this cell to be ground: the in-place
  // sequential pass and this two-phase (decide, then apply) pass are identical.  Own channels only.
  {
    float newh[kCellsPerThread];
    unsigned flip = 0;
#pragma unroll
    for (int j = 0; j < kCellsPerThread; ++j) {
      const int l = tid + j * kFusedThreads;
      newh[j] = 0.f;
      if (l < n_cells) {
        const int lc = l / kNumBin, b = l - lc * kNumBin, ch = ch0 + lc;
        if (lc >= 1 && lc <= n_own && ch >= 1 && ch < kNumChannel - 1 && b >= 1 && b < kNumBin - 1 && !G[l] && G[l + 1] &&
            G[l - 1] && G[l + kNumBin] && G[l - kNumBin]) {
          const float a = H[l + 1], bb = H[l - 1], c = H[l + kNumBin], d = H[l - kNumBin];
          const float lo1 = fminf(a, bb), hi1 = fmaxf(a, bb), lo2 = fminf(c, d), hi2 = fmaxf(c, d);
          const float m1 = fmaxf(lo1, lo2), m2 = fminf(hi1, hi2);  // the two middle values of the sorted four
          newh[j] = fdiv(fadd(m1, m2), 2.f);
          flip |= 1u << j;
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kCellsPerThread; ++j)
      if (flip & (1u << j)) { const int l = tid + j * kFusedThreads; H[l] = newh[j]; G[l] = 1; }
  }
  __syncthreads();

  // (a8) outlierFilter, ground_removal.cpp:149-174: in place along bin, so cell b sees the value written at b-1.
  // With T = tHmin, a cell is rewritten iff  A(b): all of b-1..b+2 ground, H[b]==T and (H[b+1]!=T or H[b+2]!=T),
  // and its left value is not T -- either originally, or because b-1 was itself rewritten.  Two consecutive rewrites
  // force H[b-1]==H[b]==T and H[b+1]!=T, which rules out a rewrite at b-2 (its b+2 is H[b]==T, its b+1 is T): the chain
  // is at most two cells long, so every cell's final value is a closed form of the ORIGINAL H[b-2..b+2], G[b-2..b+2].
  {
    const float T = t_hmin;
    float newh[kCellsPerThread];
    unsigned mod = 0;
#pragma unroll
    for (int j = 0; j < kCellsPerThread; ++j) {
      const int l = tid + j * kFusedThreads;
      newh[j] = 0.f;
      if (l < n_cells) {
        const int lc = l / kNumBin, b = l - lc * kNumBin, ch = ch0 + lc;
        if (lc >= 1 && lc <= n_own && ch >= 1 && ch < kNumChannel - 1 && b >= 1 && b < kNumBin - 2 && G[l] && G[l + 1] &&
            G[l - 1] && G[l + 2]) {
          const float h1 = H[l - 1], h2 = H[l], h3 = H[l + 1], h4 = H[l + 2];
          if (h2 == T && (h3 != T || h4 != T)) {                  // A(b)
            float left = h1;
            bool ok = (h1 != T);
            if (!ok && b - 1 >= 1 && G[l - 2]) {                  // was b-1 rewritten?  A(b-1) with H[b]==T needs H[b+1]!=T
              const float h0 = H[l - 2];
              if (h3 != T && h0 != T) { left = fdiv(fadd(h0, h3), 2.f); ok = true; }   // b-1 took its second branch
            }
            if (ok) { newh[j] = (h3 != T) ? fdiv(fadd(left, h3), 2.f) : fdiv(fadd(left, h4), 2.f); mod |= 1u << j; }
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kCellsPerThread; ++j)
      if (mod & (1u << j)) H[tid + j * kFusedThreads] = newh[j];
  }
  __syncthreads();

  // hGround == height for every ground cell (updateGround() follows every height write of a ground cell)
#pragma unroll
  for (int j = 0; j < kCellsPerThread; ++j) {
    const int l = tid + j * kFusedThreads;
    if (l < n_cells) {
      const int lc = l / kNumBin, b = l - lc * kNumBin, ch = ch0 + lc;
      if (lc >= 1 && lc <= n_own) {
        if (o_height) o_height[ch * kNumBin + b] = H[l];
        if (o_hg) o_hg[ch * kNumBin + b] = G[l] ? H[l] : -INFINITY;
        if (o_lim) o_lim[ch * kNumBin + b] = label_limit(H[l], G[l] != 0, p.tol);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// frame-wide barrier (all CTAs of a frame co-resident).  The counter is never reset: launch k of a slot waits for
// `target` = arrivals of all earlier launches + the arrivals this barrier needs (host-side bookkeeping).

__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned target, unsigned spin_limit) {
  __syncthreads();
  if (threadIdx.x == 0) {
    // release: the CTA's writes (ordered before this thread by the barrier above) become visible before the arrival
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(bar), "r"(1u) : "memory");
    // acquire on the polling load itself: the load that sees the last arrival synchronises with every arrival before it (they
    // are read-modify-writes on one word: one release sequence) -- no separate fence on the way out
    unsigned spin = 0;
    while ((int)(ld_acquire_u32(bar) - target) < 0)
      if (spin_limit && ++spin > spin_limit) __trap();   // a lost CTA must not hang the GPU (0 = wait for ever: debuggers, MPS)
  }
  __syncthreads();
}

constexpr int kTilePts = kFusedThreads;             // 1024 points = 16 KB per TMA tile

constexpr int kMaxResTiles = 8;                     // tiles of a CTA's chunk that stay in shared memory (128 KB): 132 CTAs hold 1.08 M points
constexpr int kDescStride = 16;                     // u64 words between two CTAs' count descriptors (128 bytes)
constexpr int kLookBatch = 5;                       // 5 x 32 >= 132 CTAs: all predecessors in one batch of loads
constexpr int kMaxTiles = 16;                       // tiles per chunk (labels of a thread's points: 2 bits each in one register)
constexpr int kPendCap = 2048;                      // points of a chunk whose cell needs the exact evaluation, queued for a compact pass
constexpr unsigned kPending = 0xFFFDu;              // cell id of a queued point until that pass has run
constexpr int kKeysPerThread = (kPolarCells + kFusedThreads - 1) / kFusedThreads;   // 10: cells of the CTA's key grid per thread
// dynamic shared memory layout (bytes): fixed part (incl. the CTA's private min-z key grid), then the resident tiles, then the cell
// ids of every tile of the chunk.
constexpr int kOffBar = 0;                                                  // [kMaxResTiles] mbarriers of the tiles + [1] of the label limits
constexpr int kOffMeta = 80;                                                // [3] pending points
constexpr int kOffCnt = 128;                                                // [16][32] u32 elevated | ground << 16 per warp
constexpr int kOffWex = kOffCnt + kMaxTiles * 32 * 4;                       // [16][32] u32 exclusive inside the tile
constexpr int kOffTtot = kOffWex + kMaxTiles * 32 * 4;                      // [16] u32 tile totals
constexpr int kOffBase = kOffTtot + kMaxTiles * 4;                          // [2] u32 chunk base (elevated, ground)
constexpr int kOffPend = (kOffBase + 16 + 15) & ~15;                        // [kPendCap] u16
constexpr int kOffG = kOffPend + kPendCap * 2;                              // [1440] u8   polar-grid slice
constexpr int kOffH = (kOffG + kMaxLocCells + 127) & ~127;                  // [1440] float
constexpr int kOffKeys = (kOffH + kMaxLocCells * 4 + 127) & ~127;           // [9600] u32  min-z keys of the CTA's own points
constexpr int kOffPts = (kOffKeys + kPolarCells * 4 + 127) & ~127;          // [res_tiles][1024] float4, then [tiles][1024] u16
__host__ __device__ constexpr int fused_smem_bytes(int res_tiles, int tiles) { return kOffPts + res_tiles * kTilePts * 16 + tiles * kTilePts * 2; }
constexpr int kFusedSmem = fused_smem_bytes(kMaxResTiles, kMaxTiles);
static_assert(kFusedSmem <= 227 * 1024, "ground_fused_kernel: shared memory budget");
static_assert(kOffBar + (kMaxResTiles + 1) * 8 <= kOffMeta && kOffMeta + 3 * 4 <= kOffCnt, "ground_fused_kernel: fixed layout");
static_assert(kDenseSmem <= kFusedSmem, "the fused CCL reuses the ground kernel's shared memory");

struct FusedOut {
  uint8_t* labels;          // nullable
  float4* elev;
  float4* ground;
  uint16_t* cart;           // nullable: cartesian cell of every elevated point (fused first pass of clustering)
  unsigned* cart_once;      // nullable: bit planes of the cartesian grid (cluster.cu)
  unsigned* cart_twice;
  int* counters;
};

// one frame of a launch: CTAs [frame * ctas_per_frame, (frame + 1) * ctas_per_frame) work on it and synchronise among themselves only
struct FrameIO {
  const float4* pts;
  int n, chunk;
  unsigned* keys;           // min-z keys of this launch
  unsigned* keys_next;      // the other grid of the slot, re-armed for its next launch
  unsigned* bar;
  unsigned bar_target;
  unsigned epoch;
  unsigned long long* desc;
  float* hg;                // [9600] nullable (inspection): hGround of ground cells, -inf otherwise
  float* lim;               // [9600] label limit of every cell (label_limit): phase 2 -> phase 3
  FusedOut out;
  // fused frame path: the last CTA of the frame to finish phase 3 labels the connected components of the bit planes all of them marked
  int fuse_ccl;
  unsigned* done_ctr;       // atomicInc counter of finished CTAs (wraps to 0 at G: needs no reset)
  CclFrame ccl;
};
struct GroundBatch {
  int n_frames, ctas_per_frame;
  unsigned spin_limit;
  FrameIO f[kMaxBatch];
  float mount[kMaxBatch][3];  // ground_fused_rig_kernel: t_hmin, t_hmax, h_sensor of each frame's sensor (phase 2); unread otherwise
};

// ground_fused_lines_kernel: frame i's ground lines (lmot_set_ground_lines) -- its ground grid (nullptr: the frame's stream has them off,
// phase 2 is groundRemove's polar grid), its sensor_height and the setting's three values
struct GroundLinesFrames {
  float* gz[kMaxBatch];
  double sensor_height[kMaxBatch], max_slope[kMaxBatch], max_rmse[kMaxBatch], max_step[kMaxBatch];
};

struct LinesSrc {
  const float* z;
  __device__ float operator()(int b) const { return z[b]; }
};
struct LinesLimDst {
  float* gz; float* lim; double tol;
  __device__ void operator()(int b, float g) const { gz[b] = g; lim[b] = label_limit(g, true, tol); }
};

// phase 2 of a frame with ground lines: the CTA's own channels' min z into shared memory (H, one coalesced pass: the walk then never
// waits for L2), then warp t's first lane walks own channel own0 + t (ground_lines.cuh) and writes its ground heights and label limits.
// One channel per warp: the walks branch differently, and lanes of one warp would run each other's branches in turn.  The halo channels
// are not needed.
__device__ __forceinline__ void lines_slice(const GroundParams& p, const GroundLinesFrames& L, int frame, const unsigned* __restrict__ keys,
                                            int own0, int n_own, float* H, float* __restrict__ lim) {
  const int tid = threadIdx.x;
  for (int l = tid; l < n_own * kNumBin; l += kFusedThreads) H[l] = fkey_inv(__ldcg(&keys[own0 * kNumBin + l]));
  __syncthreads();
  const int t = tid >> 5;
  if ((tid & 31) == 0 && t < n_own) {
    const int off = (own0 + t) * kNumBin;
    ground_lines_channel(LinesSrc{H + t * kNumBin}, LinesLimDst{L.gz[frame] + off, lim + off, p.tol}, (double)p.r_min, (double)p.r_max,
                         L.sensor_height[frame], L.max_slope[frame], L.max_rmse[frame], L.max_step[frame]);
  }
}

// the fast evaluation of polar_cell(): cell id, kNoCell (certainly outside the range window) or kPending (within the guard band
// of a cell boundary, or not a number: the exact evaluation decides)
__device__ __forceinline__ unsigned polar_cell_fast(float x, float y, const GroundParams& p) {
  const float d2 = fadd(fmul(x, x), fmul(y, y));
  const float t = __fmaf_rn(d2, rsqrtf(d2), -p.r_min) * p.bin_scale;
  const float ax = fabsf(x), ay = fabsf(y);
  const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
  const float z = __fdividef(mn, mx);
  const float u = z * z;
  float a = 0.00782548263669014f;
  a = __fmaf_rn(a, u, -0.03689862787723541f);
  a = __fmaf_rn(a, u, 0.08374155312776566f);
  a = __fmaf_rn(a, u, -0.13480405509471893f);
  a = __fmaf_rn(a, u, 0.19879871606826782f);
  a = __fmaf_rn(a, u, -0.3332637548446655f);
  a = __fmaf_rn(a, u, 0.9999993443489075f);
  a = a * z;
  if (ay > ax) a = 1.57079632679489661923f - a;
  if (x < 0.f) a = 3.14159265358979323846f - a;
  if (y < 0.f) a = -a;
  const float sc = __fmaf_rn(a, (float)(kNumChannel / 6.28318530717958647692), (float)(kNumChannel / 2));
  if (t < -kBinGuard || t > (float)kNumBin + kBinGuard) return kNoCell;      // certainly outside (rMin, rMax)
  const float tf = floorf(t), cf = floorf(sc);
  const float tr = t - tf, cr = sc - cf;
  if (!(tr > kBinGuard && tr < 1.0f - kBinGuard && cr > kChanGuard && cr < 1.0f - kChanGuard)) return kPending;
  return (unsigned)((int)cf * kNumBin + (int)tf);
}

__device__ __forceinline__ void smem_min_u32(uint32_t addr, unsigned v) {
  asm volatile("red.shared.min.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// Two tiles of phase 1 (see the kernel).  FULL: both tiles exist, are resident in shared memory and hold kTilePts points each;
// PRE: the node's pre-filters are on.
template <bool FULL, bool PRE, int kClone>
__device__ __forceinline__ void bin_pair(int t0, int T, int cnt, int res_tiles, int beg, const float4* __restrict__ pts, const float4* s_pts,
                                         uint16_t* s_cell, uint64_t* s_full, unsigned* s_meta, uint16_t* s_pend, uint32_t keys_sa,
                                         const GroundParams& p) {
  const int tid = threadIdx.x, lane = tid & 31;
  float4 q[2];
  bool valid[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int t = t0 + u;
    const int li = t * kTilePts + tid;
    if (FULL) {
      valid[u] = true;
      mbar_wait(&s_full[t], 0u);
      q[u] = s_pts[li];
    } else {
      valid[u] = t < T && li < cnt;
      q[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < T) {
        if (t < res_tiles) {
          mbar_wait(&s_full[t], 0u);
          if (valid[u]) q[u] = s_pts[li];
        } else if (valid[u]) q[u] = __ldg(&pts[beg + li]);
      }
    }
  }
  unsigned c[2], key[2];
  bool pre[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    c[u] = kNoCell;
    key[u] = 0xFFFFFFFFu;
    pre[u] = false;                              // removed by the node's pre-filters (src/groundremove/main.cpp:104-112)
    if (PRE && valid[u])
      pre[u] = !(isfinite(q[u].x) && isfinite(q[u].y) && isfinite(q[u].z) && q[u].z >= p.fz0 && q[u].z <= p.fz1 &&   // PassThrough: inclusive
                 q[u].x > p.fx0 && q[u].x < p.fx1 && q[u].y > p.fy0 && q[u].y < p.fy1);                               // ConditionalRemoval: strict
    if (valid[u] && !pre[u]) {
      c[u] = polar_cell_fast(q[u].x, q[u].y, p);
      float z = q[u].z;
      if (z == 0.f) z = 0.f;                     // -0 -> +0 (`z < minZ` does not order them either)
      if (z == z) key[u] = fkey(z);              // NaN z never wins `z < minZ` (ground_removal.cpp:41)
    }
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int t = t0 + u;
    if (!FULL && t >= T) break;                  // (CTA-uniform)
    const int li = t * kTilePts + tid;
    unsigned cc = c[u];
    // the ~1.6 per mille of points that need the exact evaluation are queued and evaluated by full warps after the loop
    // (inline, their ~170 instructions ran with one or two active lanes and stalled the other 30)
    const unsigned pm = __ballot_sync(0xFFFFFFFFu, cc == kPending);
    if (pm) {
      unsigned base = 0;
      if (lane == __ffs(pm) - 1) base = atomicAdd(&s_meta[3], (unsigned)__popc(pm));
      base = __shfl_sync(0xFFFFFFFFu, base, __ffs(pm) - 1);
      if (cc == kPending) {
        const unsigned slot = base + __popc(pm & ((1u << lane) - 1u));
        if (slot < (unsigned)kPendCap) s_pend[slot] = (uint16_t)li;
        else cc = polar_cell_exact<kClone>(q[u].x, q[u].y, p);   // queue full (adversarial clouds): evaluate here
      }
    }
    s_cell[li] = (PRE && pre[u]) ? kPreFiltered : (uint16_t)cc;
    if (cc >= (unsigned)kPolarCells) cc = kNoCell;           // pending: contributes later
    const unsigned k = (cc == kNoCell) ? 0xFFFFFFFFu : key[u];
    // min z per cell into the CTA's OWN key grid in shared memory (flushed to the frame's grid once, below).  Consecutive HDL-64
    // returns fall into the same cell: a warp that holds a single cell reduces over its lanes and issues one atomic; any other
    // warp lets the shared-memory atomic unit sort it out (one instruction; the match / group-reduce / leader code this
    // replaces was ~40 instructions on ~40 % of the warps of a dense frame)
    const unsigned c0 = __shfl_sync(0xFFFFFFFFu, cc, 0);
    if (__all_sync(0xFFFFFFFFu, cc == c0)) {
      const unsigned kmin = __reduce_min_sync(0xFFFFFFFFu, k);
      if (lane == 0 && kmin != 0xFFFFFFFFu) smem_min_u32(keys_sa + c0 * 4u, kmin);
    } else if (k != 0xFFFFFFFFu) smem_min_u32(keys_sa + cc * 4u, k);
  }
}

// ONE launch per frame -- or per batch of frames (one per sensor stream), CTA groups own frames and synchronise among themselves.
// ("No second barrier" was tried: every CTA evaluating the polar grid for the channels its own points fall into, in shared
// memory.  With ring-major clouds a chunk spans most of the 80 channels, so every CTA redid most of the grid and the kernel
// issued far more instructions.  The grid is evaluated ONCE, spread over the CTAs.)
// kRig: phase 2 takes each frame's t_hmin / t_hmax / h_sensor from B.mount (a sensor rig, lmot_set_sensors) instead of p
template <bool kRig, int kClone = 0, bool kLines = false>
__device__ __forceinline__ void ground_fused_body(const GroundBatch& B, const GroundParams& p, float roi, const GroundLinesFrames* L = nullptr) {
  extern __shared__ __align__(128) unsigned char fsm[];
  const int Gf = B.ctas_per_frame;
  const int frame = blockIdx.x / Gf, cta = blockIdx.x - frame * Gf;
  const FrameIO& F = B.f[frame];
  const float4* __restrict__ pts = F.pts;
  const int n = F.n, chunk = F.chunk;
  unsigned* __restrict__ keys = F.keys;
  const FusedOut out = F.out;
  const int T_max = (chunk + kTilePts - 1) / kTilePts;                     // tiles of a full chunk (what the launch allocated for)
  const int res_tiles = T_max < kMaxResTiles ? T_max : kMaxResTiles;
  uint64_t* s_full = reinterpret_cast<uint64_t*>(fsm + kOffBar);
  unsigned* s_meta = reinterpret_cast<unsigned*>(fsm + kOffMeta);          // [3] pending points
  unsigned* s_cnt = reinterpret_cast<unsigned*>(fsm + kOffCnt);
  unsigned* s_wex = reinterpret_cast<unsigned*>(fsm + kOffWex);
  unsigned* s_ttot = reinterpret_cast<unsigned*>(fsm + kOffTtot);
  unsigned* s_base = reinterpret_cast<unsigned*>(fsm + kOffBase);
  unsigned* s_keys = reinterpret_cast<unsigned*>(fsm + kOffKeys);
  uint16_t* s_pend = reinterpret_cast<uint16_t*>(fsm + kOffPend);
  uint8_t* s_G = fsm + kOffG;
  float* s_H = reinterpret_cast<float*>(fsm + kOffH);
  float4* s_pts = reinterpret_cast<float4*>(fsm + kOffPts);
  uint16_t* s_cell = reinterpret_cast<uint16_t*>(fsm + kOffPts + res_tiles * kTilePts * 16);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long beg_ll = (long long)cta * chunk;
  const int beg = beg_ll < n ? (int)beg_ll : n;
  const int end = min(n, beg + chunk);
  const int cnt = end - beg;
  const int T = (cnt + kTilePts - 1) / kTilePts;

  // ---- phase 0: arm the TMA copies of the resident tiles; re-arm the OTHER key grid for the slot's next frame
  // (a launch chained behind the previous ground kernel of its stream -- ground_launch_batch, `chain` -- becomes resident while that
  // kernel drains: everything up to griddep_wait() touches shared memory only; the wait returns when the preceding grid has
  // completed and its writes are visible.  An ordinary launch passes through both instructions.)
  griddep_launch_dependents();
  if (tid == 0) {
    for (int t = 0; t <= kMaxResTiles; ++t) mbar_init(&s_full[t], 1);      // [kMaxResTiles]: the label limits, phase 3
    fence_mbar_init();
  }
  if (tid < 8) s_meta[tid] = 0u;
#pragma unroll
  for (int j = 0; j < kKeysPerThread; ++j) { const int k = tid + j * kFusedThreads; if (k < kPolarCells) s_keys[k] = 0xFFFFFFFFu; }
  griddep_wait();
  if (tid == 0) {
    for (int t = 0; t < T && t < res_tiles; ++t) {
      const uint32_t bytes = (uint32_t)min(kTilePts, cnt - t * kTilePts) * 16u;
      mbar_arrive_expect_tx(&s_full[t], bytes);
      bulk_copy_g2s(s_pts + t * kTilePts, pts + beg + t * kTilePts, bytes, &s_full[t]);
    }
  }
  for (int k = cta * kFusedThreads + tid; k < kPolarCells; k += Gf * kFusedThreads) F.keys_next[k] = fkey(1000.f);  // Cell::Cell(): minZ = 1000
  __syncthreads();

  // ---- phase 1: point -> polar cell, min z per cell.  Two tiles per iteration: two independent dependency chains per thread.
  // Pairs of complete resident tiles (all of a chunk but its tail) run the variant without bounds / residency / pre-filter tests.
  {
    const uint32_t keys_sa = smem_u32(s_keys);
    const int full_end = p.prefilter ? 0 : (min(cnt / kTilePts, res_tiles) & ~1);
    int t0 = 0;
    for (; t0 < full_end; t0 += 2) bin_pair<true, false, kClone>(t0, T, cnt, res_tiles, beg, pts, s_pts, s_cell, s_full, s_meta, s_pend, keys_sa, p);
    if (p.prefilter) for (; t0 < T; t0 += 2) bin_pair<false, true, kClone>(t0, T, cnt, res_tiles, beg, pts, s_pts, s_cell, s_full, s_meta, s_pend, keys_sa, p);
    else for (; t0 < T; t0 += 2) bin_pair<false, false, kClone>(t0, T, cnt, res_tiles, beg, pts, s_pts, s_cell, s_full, s_meta, s_pend, keys_sa, p);
  }
  __syncthreads();
  {
    const int np = min((int)s_meta[3], kPendCap);
    for (int i = tid; i < np; i += kFusedThreads) {
      const int li = s_pend[i];
      const float4 q = ((li >> 10) < res_tiles) ? s_pts[li] : __ldg(&pts[beg + li]);
      const unsigned cc = polar_cell_exact<kClone>(q.x, q.y, p);
      s_cell[li] = (uint16_t)cc;
      if (cc != kNoCell) {
        float z = q.z;
        if (z == 0.f) z = 0.f;
        if (z == z) atomicMin(&s_keys[cc], fkey(z));
      }
    }
  }
  __syncthreads();
  // flush: one global atomic per cell this CTA saw a point in
#pragma unroll
  for (int j = 0; j < kKeysPerThread; ++j) {
    const int k = tid + j * kFusedThreads;
    if (k < kPolarCells) { const unsigned v = s_keys[k]; if (v != 0xFFFFFFFFu) atomicMin(&keys[k], v); }
  }
  grid_barrier(F.bar, F.bar_target, B.spin_limit);

  // ---- phase 2: the polar grid, channels split over the first min(Gf, 80) CTAs of the frame (one halo channel per side recomputed)
  {
    const int gc = Gf < kNumChannel ? Gf : kNumChannel;
    if (cta < gc) {
      const int own0 = cta * kNumChannel / gc, own1 = (cta + 1) * kNumChannel / gc;
      if (kLines && L->gz[frame]) lines_slice(p, *L, frame, keys, own0, own1 - own0, s_H, F.lim);
      else if (kRig) polar_grid_slice(p, B.mount[frame][0], B.mount[frame][1], B.mount[frame][2], keys, own0, own1 - own0, s_H, s_G, (float*)nullptr,
                                 (float*)nullptr, (float*)nullptr, (float*)nullptr, F.hg, F.lim);
      else polar_grid_slice(p, p.t_hmin, p.t_hmax, p.h_sensor, keys, own0, own1 - own0, s_H, s_G, (float*)nullptr, (float*)nullptr, (float*)nullptr,
                            (float*)nullptr, F.hg, F.lim);
    }
  }
  grid_barrier(F.bar, F.bar_target + (unsigned)Gf, B.spin_limit);

  // ---- phase 3: labels (ground_removal.cpp:221-247), per-warp counts
  unsigned labs = 0;                                // 2 bits per tile: 0 dropped, 1 ground, 2 elevated
  // Long chunks: the 38 KB of label limits come into shared memory with ONE bulk copy (over the key grid, which was flushed before
  // barrier 1) -- a gather of scattered cells from L2 moves a 32-byte sector per point.  Short chunks (an HDL-64 frame over half
  // or all of the SMs) touch fewer sectors than the grid has: they gather.
  const bool stage_lim = chunk > 2 * kTilePts;      // (frame-uniform)
  if (stage_lim) {
    if (tid == 0) {
      asm volatile("fence.proxy.async;" ::: "memory");   // the limits were written through the generic proxy (other CTAs; acquired by the barrier); so was s_keys
      mbar_arrive_expect_tx(&s_full[kMaxResTiles], (uint32_t)(kPolarCells * sizeof(float)));
      bulk_copy_g2s(s_keys, F.lim, (uint32_t)(kPolarCells * sizeof(float)), &s_full[kMaxResTiles]);
    }
    const float* s_lim = reinterpret_cast<const float*>(s_keys);
    mbar_wait(&s_full[kMaxResTiles], 0u);
    for (int t = 0; t < T; ++t) {
      const int li = t * kTilePts + tid;
      int lab = 0;
      if (li < cnt) {
        const unsigned c = s_cell[li];
        if (c == kNoCell) lab = p.prefilter ? 3 : 0;
        else if (c != kPreFiltered) {
          const float z = (t < res_tiles) ? s_pts[li].z : __ldg(&pts[beg + li]).z;
          lab = (z <= s_lim[c]) ? 1 : 2;
        }
      }
      labs |= (unsigned)lab << (2 * t);
      const unsigned be = __ballot_sync(0xFFFFFFFFu, lab == 2);
      const unsigned bg = __ballot_sync(0xFFFFFFFFu, lab == 1);
      if (lane == 0) s_cnt[t * 32 + warp] = (unsigned)__popc(be) | ((unsigned)__popc(bg) << 16);
    }
  } else {
  // label limits of this thread's points in the resident tiles: all loads issued before the first is used (one L2 round trip for
  // the whole chunk instead of one per tile)
  float lv[kMaxResTiles];
#pragma unroll
  for (int t = 0; t < kMaxResTiles; ++t) {
    lv[t] = __int_as_float(0x7FC00000);
    const int li = t * kTilePts + tid;
    if (t < T && li < cnt) { const unsigned c = s_cell[li]; if (c < kPreFiltered) lv[t] = __ldcg(&F.lim[c]); }
  }
  for (int t = 0; t < T; ++t) {
    const int li = t * kTilePts + tid;
    int lab = 0;
    if (li < cnt) {
      const unsigned c = s_cell[li];
      if (c == kNoCell) lab = p.prefilter ? 3 : 0;      // in neither output; with the node pre-filters on: still an aux point
      else if (c != kPreFiltered) {
        const float z = (t < res_tiles) ? s_pts[li].z : __ldg(&pts[beg + li]).z;
        float lm;
        switch (t) {                                            // (register array: constant indices only)
          case 0: lm = lv[0]; break; case 1: lm = lv[1]; break; case 2: lm = lv[2]; break; case 3: lm = lv[3]; break;
          case 4: lm = lv[4]; break; case 5: lm = lv[5]; break; case 6: lm = lv[6]; break;
          default: lm = __ldcg(&F.lim[c]);
        }
        lab = (z <= lm) ? 1 : 2;                                // == (double)z < hGround + 0.25 on a ground cell (:236-246), see label_limit
      }
    }
    labs |= (unsigned)lab << (2 * t);
    const unsigned be = __ballot_sync(0xFFFFFFFFu, lab == 2);
    const unsigned bg = __ballot_sync(0xFFFFFFFFu, lab == 1);
    if (lane == 0) s_cnt[t * 32 + warp] = (unsigned)__popc(be) | ((unsigned)__popc(bg) << 16);
  }
  }
  __syncthreads();
  if (warp < T) {                                   // warp w scans the 32 warp counts of tile w
    const unsigned v = s_cnt[warp * 32 + lane];
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += u; }
    s_wex[warp * 32 + lane] = inc - v;
    if (lane == 31) s_ttot[warp] = inc;
  }
  __syncthreads();
  if (warp == 0) {
    // chunk totals -> published once; every CTA sums the totals of its predecessors (all CTAs of the frame are co-resident)
    unsigned te = 0, tg = 0;
    if (lane < T) { const unsigned v = s_ttot[lane]; te = v & 0xFFFFu; tg = v >> 16; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { te += __shfl_xor_sync(0xFFFFFFFFu, te, o); tg += __shfl_xor_sync(0xFFFFFFFFu, tg, o); }
    // one word per CTA: launch tag (32) | elevated (16) | ground (16); a chunk holds at most 16384 points.  The words sit
    // kDescStride apart (one 128-byte line each): with all of them in a few adjacent lines, every CTA polling the same
    // L2 slices serialised the whole exchange
    const unsigned epoch = F.epoch;
    volatile unsigned long long* d = F.desc;
    if (lane == 0) d[cta * kDescStride] = ((unsigned long long)epoch << 32) | ((unsigned long long)te << 16) | tg;
    unsigned se = 0, sg = 0;
    for (int j0 = 0; j0 < cta; j0 += 32 * kLookBatch) {      // kLookBatch independent loads in flight per lane: one L2 round trip
      unsigned long long v[kLookBatch];
#pragma unroll
      for (int q = 0; q < kLookBatch; ++q) { const int j = j0 + q * 32 + lane; v[q] = (j < cta) ? d[j * kDescStride] : ((unsigned long long)epoch << 32); }
#pragma unroll
      for (int q = 0; q < kLookBatch; ++q) {
        const int j = j0 + q * 32 + lane;
        unsigned spin = 0;
        while ((unsigned)(v[q] >> 32) != epoch) {
          v[q] = d[j * kDescStride];
          if (B.spin_limit && ++spin > B.spin_limit) __trap();
        }
        se += (unsigned)(v[q] >> 16) & 0xFFFFu; sg += (unsigned)v[q] & 0xFFFFu;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { se += __shfl_xor_sync(0xFFFFFFFFu, se, o); sg += __shfl_xor_sync(0xFFFFFFFFu, sg, o); }
    if (lane == 0) {
      s_base[0] = se; s_base[1] = sg;
      if (cta == Gf - 1) { out.counters[CNT_N_ELEV] = (int)(se + te); out.counters[CNT_N_GROUND] = (int)(sg + tg); }
    }
  }
  __syncthreads();

  // ---- phase 3b: order-preserving output clouds + the first pass of clustering on the elevated points
  unsigned run_e = s_base[0], run_g = s_base[1];
  const unsigned lt = (1u << lane) - 1u;
  for (int t = 0; t < T; ++t) {
    const int li = t * kTilePts + tid;
    const int lab = (int)((labs >> (2 * t)) & 3u);
    const unsigned be = __ballot_sync(0xFFFFFFFFu, lab == 2);
    const unsigned bg = __ballot_sync(0xFFFFFFFFu, lab == 1);
    const unsigned wex = s_wex[t * 32 + warp];
    unsigned cc = kNoCell;
    if (li < cnt) {
      if (out.labels) out.labels[beg + li] = (uint8_t)lab;
      if (lab == 1 || lab == 2) {
        const float4 q = (t < res_tiles) ? s_pts[li] : __ldg(&pts[beg + li]);
        if (lab == 2) {
          const unsigned pos = run_e + (wex & 0xFFFFu) + __popc(be & lt);
          out.elev[pos] = make_float4(q.x, q.y, q.z, 1.f);
          if (out.cart) { cc = cart_cell_of(q.x, q.y, roi, kNumGrid); out.cart[pos] = (uint16_t)cc; }
        } else {
          out.ground[run_g + (wex >> 16) + __popc(bg & lt)] = make_float4(q.x, q.y, q.z, 1.f);
        }
      }
    }
    if (out.cart_once) cart_mark(cc, out.cart_once, out.cart_twice);   // one atomic per distinct cell per warp
    const unsigned tt = s_ttot[t];
    run_e += tt & 0xFFFFu; run_g += tt >> 16;
  }

  // ---- component clustering of this frame by the last of its CTAs to get here: no launch (and no launch latency) between ground
  // removal and clustering, and the CCL of a frame that finishes early overlaps the other frames' tails (batched launches)
  if (F.fuse_ccl) {
    __shared__ int s_last;
    __threadfence();                               // the CTA's bit-plane atomics and cartesian cells are visible device-wide ...
    __syncthreads();
    if (tid == 0) s_last = (atomicInc(F.done_ctr, (unsigned)Gf - 1u) == (unsigned)Gf - 1u) ? 1 : 0;    // ... before it counts as finished
    __syncthreads();
    if (s_last) {
      __threadfence();
      ccl_dense_body(F.ccl, fsm);     // 1,024 threads, reuses the kernel's dynamic shared memory (>= kDenseSmem, see ground_launch_batch)
    }
  }
}

__global__ void __launch_bounds__(kFusedThreads, 1)
ground_fused_kernel(const __grid_constant__ GroundBatch B, const __grid_constant__ GroundParams p, float roi) { ground_fused_body<false>(B, p, roi); }

// batched ticks of a sensor rig: the same kernel with every frame's ground thresholds from its own sensor
__global__ void __launch_bounds__(kFusedThreads, 1)
ground_fused_rig_kernel(const __grid_constant__ GroundBatch B, const __grid_constant__ GroundParams p, float roi) { ground_fused_body<true>(B, p, roi); }

// sequence ticks with their own detection values (lmot_seq_set_detect_params): every frame's whole GroundParams and clustering ROI, the
// sensor's four mounting values folded in on the host.  A separate parameter block, so that GroundBatch -- and with it the parameter
// layout of the two kernels above -- stays as it was.
struct GroundFrameParams {
  GroundParams p[kMaxBatch];
  float roi[kMaxBatch];
};
static_assert(sizeof(GroundBatch) + sizeof(GroundFrameParams) <= 4096, "ground_fused_frame_kernel: parameter block");

// the same kernel with every frame's parameters from its own entry: range filter, fast path, pre-filters (phase 1), clamp, flags,
// outlier filter and label limits (phase 2), cartesian cell (phase 3)
__global__ void __launch_bounds__(kFusedThreads, 1)
ground_fused_frame_kernel(const __grid_constant__ GroundBatch B, const __grid_constant__ GroundFrameParams P) {
  const int frame = blockIdx.x / B.ctas_per_frame;
  ground_fused_body<false, 1>(B, P.p[frame], P.roi[frame]);
}

// ground lines (lmot_set_ground_lines): the per-frame kernel with phase 2 replaced by each frame's lines where its stream has them on
static_assert(sizeof(GroundBatch) + sizeof(GroundFrameParams) + sizeof(GroundLinesFrames) <= 4096, "ground_fused_lines_kernel: parameter block");
__global__ void __launch_bounds__(kFusedThreads, 1)
ground_fused_lines_kernel(const __grid_constant__ GroundBatch B, const __grid_constant__ GroundFrameParams P,
                          const __grid_constant__ GroundLinesFrames L) {
  const int frame = blockIdx.x / B.ctas_per_frame;
  ground_fused_body<false, 2, true>(B, P.p[frame], P.roi[frame], &L);
}

// inspection only (lmot_debug_polar_grid): all five 80x120 grids of the reference from the min-z keys of the last launch, ten
// channels per CTA.  (The fused kernel evaluates, per CTA, only the channels that CTA's points need, and keeps them in shared memory.)
__global__ void __launch_bounds__(kFusedThreads)
polar_grid_debug_kernel(GroundParams p, const unsigned* __restrict__ keys, float* __restrict__ o_minz, float* __restrict__ o_height,
                        float* __restrict__ o_smoothed, float* __restrict__ o_hdiff, float* __restrict__ o_hg) {
  __shared__ float s_H[kMaxLocCells];
  __shared__ uint8_t s_G[kMaxLocCells];
  const int gc = gridDim.x;
  const int own0 = blockIdx.x * kNumChannel / gc, own1 = (blockIdx.x + 1) * kNumChannel / gc;
  polar_grid_slice(p, p.t_hmin, p.t_hmax, p.h_sensor, keys, own0, own1 - own0, s_H, s_G, o_minz, o_height, o_smoothed, o_hdiff, o_hg);
}

// inspection only (lmot_debug_cell_index): the fused kernel keeps the cell ids in shared memory
__global__ void polar_cells_kernel(const float4* __restrict__ pts, int n, GroundParams p, uint16_t* __restrict__ cell) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float4 q = __ldg(&pts[i]);
    const bool pre = p.prefilter && !(isfinite(q.x) && isfinite(q.y) && isfinite(q.z) && q.z >= p.fz0 && q.z <= p.fz1 &&
                                      q.x > p.fx0 && q.x < p.fx1 && q.y > p.fy0 && q.y < p.fy1);
    cell[i] = pre ? kNoCell : polar_cell(q.x, q.y, p);
  }
}

__global__ void init_keys_kernel(unsigned* keys, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) keys[k] = fkey(1000.f);
}

}  // namespace

int ground_alloc(Ctx* c, Slot* s) {
  const size_t np = (size_t)c->max_points;
  cudaStream_t st = s->stream;
  // co-residency limit of the cooperative kernel on this device (1 CTA per SM at this shared-memory size)
  if (c->fused_max_ctas == 0) {
    LMOT_CUDA(c, cudaFuncSetAttribute(ground_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFusedSmem));
    LMOT_CUDA(c, cudaFuncSetAttribute(ground_fused_rig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFusedSmem));
    LMOT_CUDA(c, cudaFuncSetAttribute(ground_fused_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFusedSmem));
    LMOT_CUDA(c, cudaFuncSetAttribute(ground_fused_lines_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFusedSmem));
    int sms = 0, per_sm = 0, coop = 0;
    LMOT_CUDA(c, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    LMOT_CUDA(c, cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device));
    // the grid barrier needs every CTA co-resident: the limit is the smallest over the four variants a launch may pick
    const void* variants[] = {(const void*)ground_fused_kernel, (const void*)ground_fused_rig_kernel, (const void*)ground_fused_frame_kernel,
                              (const void*)ground_fused_lines_kernel};
    per_sm = INT_MAX;
    for (const void* k : variants) {
      int v = 0;
      LMOT_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k, kFusedThreads, kFusedSmem));
      if (v < per_sm) per_sm = v;
    }
    if (!coop || per_sm < 1 || sms * per_sm < kMinCtas) { c->last_error = "device cannot run the cooperative ground kernel"; return LMOT_ERR_CUDA; }
    c->fused_max_ctas = sms * per_sm;
    if ((long long)c->fused_max_ctas * kMaxTiles * kTilePts < (long long)c->max_points) {
      c->last_error = "max_points exceeds what one cooperative launch covers on this device";
      return LMOT_ERR_CAPACITY;
    }
  }
  LMOT_CUDA(c, cudaMalloc(&s->d_points, np * sizeof(float4)));
  LMOT_CUDA(c, cudaMalloc(&s->d_stage_in, np * 4 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_cell, np * sizeof(uint16_t)));
  LMOT_CUDA(c, cudaMalloc(&s->d_polar_key, 2 * kPolarCells * sizeof(unsigned)));
  LMOT_CUDA(c, cudaMalloc(&s->d_minz, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_height, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_smoothed, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_hdiff, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_hg, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_lim, kPolarCells * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_labels, np));
  LMOT_CUDA(c, cudaMalloc(&s->d_elev, np * sizeof(float4)));
  LMOT_CUDA(c, cudaMalloc(&s->d_ground, np * sizeof(float4)));
  LMOT_CUDA(c, cudaMalloc(&s->d_gdesc, (size_t)kDescStride * c->fused_max_ctas * sizeof(unsigned long long)));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_gdesc, 0, (size_t)kDescStride * c->fused_max_ctas * sizeof(unsigned long long), st));
  LMOT_CUDA(c, cudaMalloc(&s->d_gbar, 2 * sizeof(unsigned)));            // [0] barrier arrivals, [1] finished CTAs (fused CCL)
  LMOT_CUDA(c, cudaMemsetAsync(s->d_gbar, 0, 2 * sizeof(unsigned), st));
  s->bar_base = 0; s->epoch = 0;
  LMOT_CUDA(c, cudaMalloc(&s->d_counters, CNT_COUNT * sizeof(int)));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_counters, 0, CNT_COUNT * sizeof(int), st));
  LMOT_CUDA(c, cudaHostAlloc(&s->h_counters, CNT_COUNT * sizeof(int), cudaHostAllocDefault));
  LMOT_CUDA(c, cudaHostAlloc(&s->h_set, CNT_COUNT * sizeof(int), cudaHostAllocDefault));
  init_keys_kernel<<<(2 * kPolarCells + 255) / 256, 256, 0, st>>>(s->d_polar_key, 2 * kPolarCells);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

void ground_free(Slot* s) {
  cudaFree(s->d_points); cudaFree(s->d_stage_in); cudaFree(s->d_cell); cudaFree(s->d_polar_key); cudaFree(s->d_minz);
  cudaFree(s->d_height); cudaFree(s->d_smoothed); cudaFree(s->d_hdiff); cudaFree(s->d_hg); cudaFree(s->d_lim); cudaFree(s->d_hg_dbg); cudaFree(s->d_labels);
  cudaFree(s->d_elev); cudaFree(s->d_ground); cudaFree(s->d_gdesc); cudaFree(s->d_gbar); cudaFree(s->d_counters);
  if (s->h_counters) cudaFreeHost(s->h_counters);
  if (s->h_set) cudaFreeHost(s->h_set);
}

int ground_repack(Ctx* c, cudaStream_t st, const float* d_in, int n, int stride, float4* d_out) {
  if (n > 0) repack_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_in, n, stride, d_out);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// per-point polar cell ids of the slot's current frame, recomputed with the same device function (inspection only)
int ground_cells_debug(Ctx* c, Slot* s, cudaStream_t st) {
  if (s->cur_n > 0) polar_cells_kernel<<<(s->cur_n + 255) / 256, 256, 0, st>>>(s->cur_points, s->cur_n, c->gp, s->d_cell);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// does a frame of n points stay resident in shared memory in the frame pipeline's launch geometry?  (then the kernel reads every
// input byte exactly once, and the frame may be read straight from pinned host memory -- api.cu lmot_frame_submit)
bool ground_reads_input_once(const Ctx* c, int n) {
  int cap = c->fused_max_ctas;
  if (c->ground_half_sms) { const int half = cap / 2 > kMinCtas ? cap / 2 : kMinCtas; if ((long long)half * kMaxResTiles * kTilePts >= (long long)n) cap = half; }
  return (long long)cap * kMaxResTiles * kTilePts >= (long long)n;
}

// One launch for F frames (F = 1: the frame pipeline and the stage entry points; F > 1: one frame per sensor stream, api.cu
// lmot_batch_*).  Frame i runs on slots[i]'s buffers; its CTAs are [i * G, (i + 1) * G) of the grid and synchronise among themselves.
int ground_launch_batch(Ctx* c, Slot* const* slots, int F, const float4* const* pts, const int* n, cudaStream_t st, bool fuse_count,
                        bool want_labels, bool fuse_ccl, bool chain, const lmot_sensor* rig, const lmot_detect_params* det,
                        const GroundLinesJob* lines) {
  if (fuse_ccl && !fuse_count) return LMOT_ERR_INVALID;
  if (F < 1 || F > kMaxBatch) return LMOT_ERR_INVALID;
  int n_max = 0;
  for (int i = 0; i < F; ++i) { slots[i]->cur_points = pts[i]; slots[i]->cur_n = n[i]; if (n[i] > n_max) n_max = n[i]; }
  // CTAs per frame: enough that a chunk is a handful of 16 KB tiles, never more than can be co-resident
  int G = (n_max + c->pts_per_cta - 1) / c->pts_per_cta;
  if (G < kMinCtas) G = kMinCtas;
  int cap = c->fused_max_ctas / F;
  // Inside the frame pipeline the kernel keeps to HALF of the SMs (as long as its chunks still fit in shared memory): a
  // 1024-thread CTA holds 48 K of an SM's 64 K registers, and with the box-fitting CTAs of another frame next to it the SM has no
  // room for a CTA of the tracker chain -- the last imm_predict_gate CTA then starts well after the first one and stretches the
  // sequential chain (the bound of frames/s).  Detection has slack per frame.
  if (F == 1 && fuse_count && c->ground_half_sms) {
    const int half = cap / 2 > kMinCtas ? cap / 2 : kMinCtas;
    if ((long long)half * kMaxResTiles * kTilePts >= (long long)n_max) cap = half;
  }
  if (cap < 1) return LMOT_ERR_CAPACITY;
  if (G > cap) G = cap;
  GroundBatch B;
  memset(&B, 0, sizeof(B));
  B.n_frames = F; B.ctas_per_frame = G; B.spin_limit = c->spin_limit;
  int chunk_max = 0;
  for (int i = 0; i < F; ++i) {
    Slot* s = slots[i];
    FrameIO& f = B.f[i];
    f.pts = pts[i]; f.n = n[i];
    f.chunk = (n[i] + G - 1) / G;
    if (f.chunk > kMaxTiles * kTilePts) return LMOT_ERR_CAPACITY;
    if (f.chunk > chunk_max) chunk_max = f.chunk;
    const int parity = (int)(s->epoch & 1u);
    s->epoch += 1;
    f.keys = s->d_polar_key + parity * kPolarCells;
    f.keys_next = s->d_polar_key + (1 - parity) * kPolarCells;
    f.bar = s->d_gbar; f.bar_target = s->bar_base + (unsigned)G;
    f.hg = want_labels ? s->d_hg : nullptr; f.lim = s->d_lim;
    f.fuse_ccl = fuse_ccl ? 1 : 0; f.done_ctr = s->d_gbar + 1;
    f.ccl.once = s->d_cart_bits; f.ccl.twice = s->d_cart_bits + 2000; f.ccl.prev_occ = s->d_cart_bits + 4000;
    f.ccl.out = s->d_label_grid; f.ccl.counters = s->d_counters;
    s->hg_valid = want_labels;
    f.epoch = s->epoch; f.desc = s->d_gdesc;
    f.out.labels = want_labels ? s->d_labels : nullptr;
    f.out.elev = s->d_elev; f.out.ground = s->d_ground;
    f.out.cart = fuse_count ? s->d_cart : nullptr;
    f.out.cart_once = fuse_count ? s->d_cart_bits : nullptr;
    f.out.cart_twice = fuse_count ? s->d_cart_bits + 2000 : nullptr;
    f.out.counters = s->d_counters;
    s->bar_base += 2u * (unsigned)G;
  }
  if (rig)
    for (int i = 0; i < F; ++i) { B.mount[i][0] = rig[i].t_hmin; B.mount[i][1] = rig[i].t_hmax; B.mount[i][2] = rig[i].h_sensor; }
  const void* kern = det ? (const void*)ground_fused_frame_kernel : rig ? (const void*)ground_fused_rig_kernel : (const void*)ground_fused_kernel;
  float roi = c->prm.roi_m;
  GroundParams gp = c->gp;
  void* args3[] = {(void*)&B, (void*)&gp, (void*)&roi};
  GroundFrameParams FP;
  void* args2[] = {(void*)&B, (void*)&FP};
  GroundLinesFrames L;
  memset(&L, 0, sizeof(L));
  void* argsl[] = {(void*)&B, (void*)&FP, (void*)&L};
  if (det || lines) {
    memset(&FP, 0, sizeof(FP));
    const lmot_detect_params base = detect_params_of(c->prm);
    for (int i = 0; i < F; ++i) {
      lmot_detect_params d = det ? det[i] : base;
      if (!det && rig) { d.h_sensor = rig[i].h_sensor; d.t_hmin = rig[i].t_hmin; d.t_hmax = rig[i].t_hmax; d.sensor_height = rig[i].sensor_height; }
      FP.p[i] = ground_params_of(d, c->gp.tap); FP.roi[i] = d.roi_m;
      if (lines) {
        const lmot_ground_lines* g = lines[i].cfg;
        L.gz[i] = g ? lines[i].gz : nullptr;
        L.sensor_height[i] = d.sensor_height;
        if (g) { L.max_slope[i] = g->max_slope; L.max_rmse[i] = g->max_rmse; L.max_step[i] = g->max_step; }
      }
    }
  }
  if (lines) kern = (const void*)ground_fused_lines_kernel;
  void** args = lines ? argsl : det ? args2 : args3;
  // every frame's chunk is laid out with the tile count of the longest one (the kernel derives its layout from its own chunk;
  // a shorter chunk just leaves the tail of the allocation unused)
  const int tiles = (chunk_max + kTilePts - 1) / kTilePts;
  size_t smem = (size_t)fused_smem_bytes(tiles < kMaxResTiles ? tiles : kMaxResTiles, tiles > 0 ? tiles : 1);
  if (fuse_ccl && smem < (size_t)kDenseSmem) smem = kDenseSmem;
  if (c->coop_launch) {
    LMOT_CUDA(c, cudaLaunchCooperativeKernel(kern, dim3(G * F), dim3(kFusedThreads), args, smem, st));
  } else {
    // Ordinary launch + the guarantee a cooperative launch would give, obtained differently.  A cooperative launch makes
    // the driver wait for an idle device, i.e. it serialises the frame pipeline's streams (measured: the detection stages of
    // different frames stopped overlapping).  The kernel's barrier only needs all G * F CTAs to BECOME resident: G * F <= one
    // CTA per SM (fused_max_ctas), every other kernel on the device terminates without waiting for this one, and ground
    // kernels never wait for each other because they are chained through one per-device event -- at most one is in flight,
    // so no two partially resident grids can starve each other.  (Several PROCESSES sharing the GPU through MPS are outside
    // this guarantee; the barrier then traps after `spin_limit` polls instead of hanging -- LMOT_SPIN_LIMIT=0 waits for ever.)
    std::lock_guard<std::mutex> lk(g_ground_mutex);
    GroundChain& g = g_chain[c->device & 63];
    if (!g.done) LMOT_CUDA(c, cudaEventCreateWithFlags(&g.done, cudaEventDisableTiming));
    const bool same_stream = g.have_last && g.last == st;
    if (!same_stream) {
      if (g.record_pending) {
        // (a caller stream that was destroyed without lmot_set_stream: its work still runs to completion -- wait for the device instead)
        if (cudaEventRecord(g.done, g.last) == cudaSuccess) g.recorded = true;
        else { cudaGetLastError(); LMOT_CUDA(c, cudaDeviceSynchronize()); }
        g.record_pending = false;
      }
      if (g.recorded) LMOT_CUDA(c, cudaStreamWaitEvent(st, g.done, 0));
    }
    // chained behind a ground kernel on the same stream: programmatic dependent launch -- this grid's CTAs become resident and set
    // up their shared memory while the previous grid drains (its fused clustering tail included), see the kernel's griddep_wait()
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(G * F); cfg.blockDim = dim3(kFusedThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (chain && same_stream && g.record_pending && !c->timing) ? 1 : 0;
    LMOT_CUDA(c, cudaLaunchKernelExC(&cfg, kern, args));
    if (chain) g.record_pending = true;
    else { LMOT_CUDA(c, cudaEventRecord(g.done, st)); g.record_pending = false; g.recorded = true; }
    g.last = st; g.have_last = true;
  }
  kernel_mark(c, slots[0], st);
  return LMOT_OK;
}

int ground_launch(Ctx* c, Slot* s, cudaStream_t st, const float4* pts, int n, bool fuse_count, bool want_labels, bool fuse_ccl, bool chain) {
  Slot* sl[1] = {s};
  const float4* pp[1] = {pts};
  const int nn[1] = {n};
  return ground_launch_batch(c, sl, 1, pp, nn, st, fuse_count, want_labels, fuse_ccl, chain);
}

// a stream is about to go away.  Caller's stream replaced (lmot_set_stream; the old one is still valid): record what a later launch
// on another stream would have recorded on it.  Context destroyed after a device-wide synchronise (`device_idle`): nothing is left
// to wait for, and the stream handle may already be stale -- just drop it.
void ground_chain_forget(int device, bool device_idle) {
  std::lock_guard<std::mutex> lk(g_ground_mutex);
  GroundChain& g = g_chain[device & 63];
  if (g.record_pending && g.done && !device_idle) {
    if (cudaEventRecord(g.done, g.last) == cudaSuccess) g.recorded = true;
    else cudaGetLastError();
  }
  g.record_pending = false;
  g.have_last = false;
}

// all five polar grids of the slot's LAST ground launch, recomputed from its min-z keys (inspection only)
int ground_grids_debug(Ctx* c, Slot* s, cudaStream_t st) {
  if (s->epoch == 0) return LMOT_ERR_STATE;
  if (!s->d_hg_dbg) LMOT_CUDA(c, cudaMalloc(&s->d_hg_dbg, kPolarCells * sizeof(float)));
  const unsigned* keys = s->d_polar_key + ((s->epoch - 1u) & 1u) * kPolarCells;
  polar_grid_debug_kernel<<<kMinCtas, kFusedThreads, 0, st>>>(c->gp, keys, s->d_minz, s->d_height, s->d_smoothed, s->d_hdiff, s->d_hg_dbg);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace lmot
