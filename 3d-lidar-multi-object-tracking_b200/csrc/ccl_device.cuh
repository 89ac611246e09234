// ccl_device.cuh -- connected components of the 250x250 occupancy bitmap by ONE CTA of 1,024 threads, as a device function:
// cluster.cu wraps it in ccl_dense_kernel (one CTA per frame), ground.cu calls it from the last CTA of a frame to finish
// (fused frame path: no launch between ground removal and clustering).  See cluster.cu for the algorithm's description.
#pragma once
#include "lmot_internal.cuh"

namespace lmot {

constexpr int kRowWords = 8;                                   // 250 bits per row
constexpr int kBitWords = kNumGrid * kRowWords;                // 2000
constexpr unsigned kLastWordMask = (1u << (kNumGrid - 32 * (kRowWords - 1))) - 1u;   // bits 0..25 of word 7
constexpr int kPiecesPerWord = 16;
constexpr int kNodes = kBitWords * kPiecesPerWord;             // 32000
constexpr int kCclThreads = 1024;

// ---- union-find over shared-memory nodes, root = smallest id -------------------------------------------------
// find with path halving: every visited node is re-pointed at its grandparent.  Parents only ever move to an ancestor
// (a smaller id), so concurrent finds / unions by other threads stay correct, and the chains that the row-by-row links
// would otherwise build (one hop per grid row of a tall component) collapse while the unions are still being made.
__device__ __forceinline__ int uf_find(volatile int* L, int x) {
  int p = L[x];
  while (p != x) {
    const int g = L[p];
    if (g != p) L[x] = g;
    x = p; p = g;
  }
  return x;
}

// read-only find for the flattening pass: there, the only writes are final roots (a halving store by another thread could
// land after the owner's flattening store and point the node back at an intermediate ancestor)
__device__ __forceinline__ int uf_root(const volatile int* L, int x) {
  int p = L[x];
  while (p != x) { x = p; p = L[x]; }
  return x;
}

__device__ __forceinline__ void uf_union(volatile int* L, int* Lw, int a, int b) {
  while (true) {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&Lw[b], a);
    if (old == b) return;
    b = old;
  }
}

// horizontal 3-tap dilation of one word of a row (neighbour words supply the carry bits)
__device__ __forceinline__ unsigned hdil(const unsigned* row, int k) {
  const unsigned s = row[k];
  unsigned d = s | (s << 1) | (s >> 1);
  if (k > 0) d |= row[k - 1] >> 31;
  if (k < kRowWords - 1) d |= row[k + 1] << 31;
  return d;
}

__device__ __forceinline__ unsigned piece_starts(unsigned m) { return m & ~(m << 1); }
// index (inside its word) of the piece that contains set bit p of word m
__device__ __forceinline__ int piece_of(unsigned m, int p) { return __popc(piece_starts(m) & ((2u << p) - 1u)) - 1; }

// detection areas: whether cell c (x*250+y, or kNoCell) of a point has its bit set in the unit's cell mask
__device__ __forceinline__ bool area_kept(const unsigned* __restrict__ area, unsigned c) {
  if (c == kNoCell) return false;
  const unsigned x = c / (unsigned)kNumGrid, y = c - x * (unsigned)kNumGrid;
  return (__ldg(&area[x * kRowWords + (y >> 5)]) >> (y & 31u)) & 1u;
}

// One frame of a launch (blockIdx.x): bit planes in, label grid + cluster count out
struct CclFrame {
  unsigned* once; unsigned* twice; unsigned* prev_occ;
  int* out;
  int* counters;
};
struct CclBatch { CclFrame f[kMaxBatch]; };

// pointer jumping: re-point x at its grandparent until its parent is a root.  Only the owner of x stores to L[x] here and every
// store moves x to an ancestor, so the walks of all threads run concurrently and shorten each other: a chain of n pieces
// (a tall object: one link per grid row) collapses in ~log2(n) rounds instead of n dependent loads per thread.
__device__ __forceinline__ int uf_compress(volatile int* L, int x) {
  int p = L[x];
  while (true) {
    const int g = L[p];
    if (g == p) break;
    L[x] = g;
    p = g;
  }
  return p;
}

// ---------------------------------------------------------------------------------------------------------------
// Node ids are DENSE.  (Round 1 / the first version of round 2 numbered a piece word * 16 + k: the 32 lanes of a warp then hit the
// same shared-memory bank on every parent access, each thread walked its own ragged list of pieces, and every flatten / union was a
// data-dependent loop of dependent loads.)  A block-wide scan of the pieces per word gives every piece its
// raster-order rank as id (still monotone: the smallest id of a component is its first piece in raster order), so that
//   * flattening is pointer jumping with thread t on ids t, t + 1024, ...: conflict-free, ~log2(depth) steps per node;
//   * the adjacencies step C cannot express as a parent link go to a pair list and are united one pair per thread.
constexpr int kPairCap = 4096;
constexpr int kDenseSmem = kNodes * 4 + 3 * kBitWords * 4 + (kBitWords + 8) * 4 + kPairCap * 4 + 64 * 4;

// flatten: every node re-points itself at its grandparent until its parent is a root (uf_compress), thread t on ids t, t + 1024,
// ...; only the owner stores to L[id], every store moves id to an ancestor, roots do not change while this runs -- so the walks
// need no barrier between them and shorten each other: ~log2(depth) steps per node.  (Barrier-synchronised rounds with
// __syncthreads_or pay a CTA barrier PER ROUND.)
__device__ __forceinline__ void ccl_flatten(volatile int* L, int P) {
  for (int id = threadIdx.x; id < P; id += kCclThreads) uf_compress(L, id);
  __syncthreads();
}

// kArea: the unit's cell mask (detection areas, nullptr: every cell) is ANDed into the seeds as they load -- a masked cell holds no point
// of the masked cloud, and seeds are "more than one point per cell", so masking whole cells is exact
template <bool kArea = false>
__device__ __forceinline__ void ccl_dense_body(const CclFrame& F, unsigned char* ccl_smem, const unsigned* __restrict__ area = nullptr) {
  int* s_par = reinterpret_cast<int*>(ccl_smem);                       // [<= 32000] parent id, later -(cluster id) at roots
  unsigned* s_seed = reinterpret_cast<unsigned*>(s_par + kNodes);       // [2000]
  unsigned* s_occ = s_seed + kBitWords;                                 // [2000]
  unsigned* s_prev = s_occ + kBitWords;                                 // [2000]
  int* s_wbase = reinterpret_cast<int*>(s_prev + kBitWords);            // [2000 + 1] id of the first piece of every word
  unsigned* s_pairs = reinterpret_cast<unsigned*>(s_wbase + kBitWords + 8);   // [kPairCap] a | b << 16
  int* s_warp = reinterpret_cast<int*>(s_pairs + kPairCap);             // [32] + total, [40] pair count
  unsigned* __restrict__ once = F.once; unsigned* __restrict__ twice = F.twice; unsigned* __restrict__ prev_occ = F.prev_occ;
  int* __restrict__ out = F.out;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int w0 = 2 * tid;
  const bool own = tid < kBitWords / 2;
  // A: seed = cells with more than one point (component_clustering.cpp:136); the bit planes are re-armed for the next frame
  if (own) {
    uint2 tw = __ldcg(reinterpret_cast<const uint2*>(twice) + tid);
    if (kArea && area) { const uint2 am = __ldg(reinterpret_cast<const uint2*>(area) + tid); tw.x &= am.x; tw.y &= am.y; }
    const uint2 pv = __ldcg(reinterpret_cast<const uint2*>(prev_occ) + tid);
    s_seed[w0] = tw.x; s_seed[w0 + 1] = tw.y;
    s_prev[w0] = pv.x; s_prev[w0 + 1] = pv.y;
    reinterpret_cast<uint2*>(once)[tid] = make_uint2(0u, 0u);
    reinterpret_cast<uint2*>(twice)[tid] = make_uint2(0u, 0u);
  }
  if (tid == 0) s_warp[40] = 0;
  __syncthreads();
  // B: occupied = seed dilated 3x3, clipped at the border (:137-214); ids: exclusive scan of the pieces per word
  unsigned occ[2] = {0u, 0u};
  int np0 = 0, np1 = 0;
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned o = hdil(s_seed + x * kRowWords, k);
      if (x > 0) o |= hdil(s_seed + (x - 1) * kRowWords, k);
      if (x < kNumGrid - 1) o |= hdil(s_seed + (x + 1) * kRowWords, k);
      if (k == kRowWords - 1) o &= kLastWordMask;
      occ[h] = o;
      s_occ[w] = o;
    }
    reinterpret_cast<uint2*>(prev_occ)[tid] = make_uint2(occ[0], occ[1]);
    np0 = __popc(piece_starts(occ[0])); np1 = __popc(piece_starts(occ[1]));
  }
  int P;
  {
    const int cnt = np0 + np1;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int v = s_warp[lane];
      int wi = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += t; }
      s_warp[lane] = wi - v;
      if (lane == 31) s_warp[32] = wi;
    }
    __syncthreads();
    const int base = s_warp[warp] + incl - cnt;
    if (own) { s_wbase[w0] = base; s_wbase[w0 + 1] = base + np0; }
    P = s_warp[32];
  }
  __syncthreads();
  // C: first parent = the smallest neighbour a piece touches (leftmost touching piece of the row above, else the piece it
  // continues from the previous word, else itself); every OTHER adjacency becomes a pair for step E
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const unsigned m = occ[h];
      if (!m) continue;
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned up = 0u, upl = 0u, upr = 0u;
      int bu = 0, bul = 0, bur = 0;
      if (x > 0) {
        up = s_occ[w - kRowWords]; bu = s_wbase[w - kRowWords];
        if (k > 0) { upl = s_occ[w - kRowWords - 1]; bul = s_wbase[w - kRowWords - 1]; }
        if (k < kRowWords - 1) { upr = s_occ[w - kRowWords + 1]; bur = s_wbase[w - kRowWords + 1]; }
      }
      const unsigned left = (k > 0) ? ((h == 1) ? occ[0] : s_occ[w - 1]) : 0u;
      const int bl = (k > 0) ? s_wbase[w - 1] : 0;
      const int mybase = s_wbase[w];
      unsigned rest = m;
      int j = 0;
      while (rest) {
        const int a = __ffs(rest) - 1;
        const unsigned t = ~(rest >> a);                       // first zero above a ends the piece
        const int len = t ? __ffs(t) - 1 : 32;
        const unsigned pm = (len >= 32 ? 0xFFFFFFFFu : ((1u << len) - 1u)) << a;
        rest &= ~pm;
        const int me = mybase + j;
        ++j;
        // neighbours in DEcreasing id order; the last one found is the parent, the others go to the pair list
        int par = me;
        auto link = [&](int nb) {
          if (par != me) {                                     // the previous candidate loses: remember it as a pair
            const int slot = atomicAdd(&s_warp[40], 1);
            if (slot < kPairCap) s_pairs[slot] = (unsigned)me | ((unsigned)par << 16);   // (list full: step E re-derives ALL adjacencies instead)
          }
          par = nb;
        };
        if (a == 0 && (left >> 31)) link(bl + __popc(piece_starts(left)) - 1);                 // same row, previous word
        if (a + len == 32 && (upr & 1u)) link(bur);                                             // row above, word to the right
        unsigned touched = up & (pm | (pm << 1) | (pm >> 1));                                   // row above, same word: right to left
        while (touched) {
          const int p = 31 - __clz(touched);
          const int q = piece_of(up, p);
          link(bu + q);
          // clear this whole piece from `touched`: all bits from its start upwards
          const unsigned startbit = piece_starts(up) & ((2u << p) - 1u);                       // starts at or below p
          const int sb = 31 - __clz(startbit);                                                  // the start of the piece containing p
          touched &= (1u << sb) - 1u;
        }
        if (a == 0 && (upl >> 31)) link(bul + __popc(piece_starts(upl)) - 1);                   // row above, word to the left
        s_par[me] = par;
      }
    }
  }
  __syncthreads();
  volatile int* Lv = s_par;
  // D: flatten
  ccl_flatten(Lv, P);
  // E: the remaining adjacencies, one pair per thread
  if (s_warp[40] <= kPairCap) {
    const int npairs = s_warp[40];
    for (int i = tid; i < npairs; i += kCclThreads) { const unsigned pr = s_pairs[i]; uf_union(Lv, s_par, (int)(pr & 0xFFFFu), (int)(pr >> 16)); }
  } else if (own) {
    // more pairs than the list holds (checkerboard-like occupancy): every thread unites ALL adjacencies of its own pieces
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const unsigned m = occ[h];
      if (!m) continue;
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned up = 0u, upl = 0u, upr = 0u;
      int bu = 0, bul = 0, bur = 0;
      if (x > 0) {
        up = s_occ[w - kRowWords]; bu = s_wbase[w - kRowWords];
        if (k > 0) { upl = s_occ[w - kRowWords - 1]; bul = s_wbase[w - kRowWords - 1]; }
        if (k < kRowWords - 1) { upr = s_occ[w - kRowWords + 1]; bur = s_wbase[w - kRowWords + 1]; }
      }
      const unsigned left = (k > 0) ? ((h == 1) ? occ[0] : s_occ[w - 1]) : 0u;
      const int bl = (k > 0) ? s_wbase[w - 1] : 0;
      unsigned rest = m;
      int me = s_wbase[w];
      while (rest) {
        const int a = __ffs(rest) - 1;
        const unsigned t = ~(rest >> a);
        const int len = t ? __ffs(t) - 1 : 32;
        const unsigned pm = (len >= 32 ? 0xFFFFFFFFu : ((1u << len) - 1u)) << a;
        rest &= ~pm;
        if (a == 0 && (left >> 31)) uf_union(Lv, s_par, me, bl + __popc(piece_starts(left)) - 1);
        if (a + len == 32 && (upr & 1u)) uf_union(Lv, s_par, me, bur);
        unsigned touched = up & (pm | (pm << 1) | (pm >> 1));
        while (touched) {
          const int p = 31 - __clz(touched);
          uf_union(Lv, s_par, me, bu + piece_of(up, p));
          const unsigned startbit = piece_starts(up) & ((2u << p) - 1u);
          touched &= (1u << (31 - __clz(startbit))) - 1u;
        }
        if (a == 0 && (upl >> 31)) uf_union(Lv, s_par, me, bul + __popc(piece_starts(upl)) - 1);
        ++me;
      }
    }
  }
  __syncthreads();
  // F: flatten again
  ccl_flatten(Lv, P);
  // G: id = 1 + rank of the root among all roots in id (= raster) order (:247-257); thread t ranks the ids [t*c, (t+1)*c)
  {
    const int c = (P + kCclThreads - 1) / kCclThreads;
    const int i0 = min(tid * c, P), i1 = min(i0 + c, P);
    int roots = 0;
    for (int id = i0; id < i1; ++id) roots += (s_par[id] == id) ? 1 : 0;
    int incl = roots;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int v = s_warp[lane];
      int wi = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += t; }
      s_warp[lane] = wi - v;
      if (lane == 31) F.counters[CNT_NUM_CLUSTER] = wi;
    }
    __syncthreads();
    int rank = s_warp[warp] + incl - roots;
    // (every non-root points at its root after F, so turning roots into -(id) cannot confuse a concurrent reader: nobody reads
    // parents between here and the barrier below)
    for (int id = i0; id < i1; ++id) if (s_par[id] == id) s_par[id] = -(++rank);
  }
  __syncthreads();
  // H: label grid, sparse: cells occupied now get their id, cells occupied only in the previous frame are cleared
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h;
      const unsigned m = occ[h];
      int* o = out + (w >> 3) * kNumGrid + (w & 7) * 32;
      unsigned gone = s_prev[w] & ~m;
      while (gone) { const int b = __ffs(gone) - 1; gone &= gone - 1; o[b] = 0; }
      unsigned rest = m;
      int id = s_wbase[w];
      while (rest) {
        const int a = __ffs(rest) - 1;
        const unsigned t = ~(rest >> a);
        const int len = t ? __ffs(t) - 1 : 32;
        rest &= ~((len >= 32 ? 0xFFFFFFFFu : ((1u << len) - 1u)) << a);
        int r = s_par[id];
        ++id;
        if (r >= 0) r = s_par[r];                               // non-root: its root holds -(id)
        for (int b = a; b < a + len; ++b) o[b] = -r;
      }
    }
  }
}


}  // namespace lmot
