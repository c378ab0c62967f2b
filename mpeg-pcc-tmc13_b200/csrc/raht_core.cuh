// raht_core.cuh — the per-item bodies of the RAHT kernels.
//
// CUDA (H100, sm_90a) re-design of TMC13's region-adaptive hierarchical transform
// (tmc3/RAHT.cpp:977-1976, intra mode).  The reference reduces the Morton
// sorted voxel list one binary level at a time into LF/HF vectors and then
// re-expands it while transforming (a single sequential walk).  Here every
// transform stage (each third binary level that adds nodes) is materialised
// once in HBM as a structure-of-arrays node list in Morton order; all
// bottom-up work (duplicate merge, weights, wrapping int32 sums, qp
// averages) is data-parallel over nodes, and the top-down pass is
// data-parallel over blocks of siblings, ordered only by the true
// dependencies of the algorithm:
//   * a block reads the current-stage reconstruction of those of its 12
//     face/edge neighbour blocks that precede it in Morton order
//     (sub-node prediction, RAHT.cpp:370-415,503-565), and
//   * the encoder's RDOQ zero-run counter is carried through all
//     coefficients in coding order (RAHT.cpp:1154,1618-1669).
// Both are resolved on the device by per-block ready flags (spin on an
// earlier block's flag; a decoupled look-back for the zero-run counter).
//
// Every functor below is `__host__ __device__` so that the same bodies run
// as CUDA kernels (exec_cuda.cuh) and, for the CPU unit tests only, as plain
// loops (tests/emu).
#pragma once

#include "pcc_arith.cuh"

namespace pccb200 {

//============================================================================
// memory-ordering helpers for the block-level dataflow

#if defined(__CUDA_ARCH__)
PCC_HD int
ld_acquire(const int* p)
{
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
PCC_HD void
st_release(int* p, int v)
{
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
PCC_HD void
spin_pause()
{
  __nanosleep(20);
}
#else
PCC_HD int
ld_acquire(const int* p)
{
  return *p;
}
PCC_HD void
st_release(int* p, int v)
{
  *p = v;
}
PCC_HD void
spin_pause()
{
}
#endif

template<class T>
PCC_HD void
atomic_add_i32(T* p, T v)
{
#if defined(__CUDA_ARCH__)
  atomicAdd(p, v);
#else
  *p += v;
#endif
}

PCC_HD void
atomic_or_i32(int* p, int v)
{
#if defined(__CUDA_ARCH__)
  atomicOr(p, v);
#else
  *p |= v;
#endif
}

//============================================================================
// one transform stage in HBM (structure of arrays, Morton order)

struct Stage {
  int level;         // nodes are unique in (key >> level)
  int n;             // node count
  int64_t* key;      // Morton code of the node's first leaf
  int32_t* weight;   // number of points below the node
  int32_t* attr;     // n*A  attribute sums (int32, wrapping) or Haar low-pass
  int32_t* qpUp;     // n*2  region qp offset << 4 averaged over the subtree
  int32_t* qpDown;   // n*2  the qp the node carries during the descent
  int32_t* first;    // n+1  first child in the next finer stage
  int32_t* nn;       // n    neighbour count inherited by the node's block
  uint8_t* occ;      // n    occupancy of the node's children
  int64_t* rec;      // n*A  reconstruction scaled by 1/sqrt(w)  (attrRec)
  int64_t* recUs;    // n*A  un-scaled reconstruction            (attrRecUs)
  int* done;         // n    block-of-children finished (dataflow flag)
};

// flattened parameters every kernel needs
struct RahtConfig {
  int A;
  int isEncoder;
  int ext;
  int haar;
  int hasQp;  // per-point qp offsets present
  int predictionEnabled;
  int subnode;
  int thr0, thr1;
  int searchRange;
  int predWeightParent[19];
  int predWeightChild[12];
  int numLayers;
  int maxQp;
  int fixedPointQpOffset;
  int numAcLayers;
};

// tables that do not fit kernel-argument space comfortably live in HBM
struct QpTables {
  int32_t layers[PCCB200_MAX_QP_LAYERS][2];
  int32_t acQps[PCCB200_MAX_AC_QP_LAYERS][7][2];
};

//============================================================================
// step 1: adjacent-key statistics.  hist[h] counts adjacent pairs whose
// highest differing key bit is h; hist[64] is an error word (bit 0: keys not
// ascending).  From it the host derives the leaf count and the node count of
// every level without further synchronisation.

struct LevelHistFn {
  const int64_t* key;
  int* hist;
  PCC_HD void operator()(int64_t i) const
  {
    if (i == 0)
      return;
    int64_t a = key[i - 1], b = key[i];
    if (b < a) {
      atomic_or_i32(&hist[64], 1);
      return;
    }
    uint64_t x = uint64_t(a ^ b);
    if (!x)
      return;
    const int bin = 63 - clz64(x);
#if defined(__CUDA_ARCH__)
    // adjacent keys mostly differ in the same few low bits: one atomic per bin
    // and warp instead of one per point (a million atomics on ~20 words)
    const unsigned peers = __match_any_sync(__activemask(), bin);
    if ((threadIdx.x & 31) == __ffs(peers) - 1)
      atomicAdd(&hist[bin], __popc(peers));
#else
    atomic_add_i32(&hist[bin], 1);
#endif
  }
};

//============================================================================
// head predicates / emitters for the stream compactions that build a stage

struct LeafHead {
  const int64_t* key;
  PCC_HD bool operator()(int64_t i) const { return i == 0 || key[i] != key[i - 1]; }
};

struct StageHead {
  const int64_t* key;
  int shift;
  PCC_HD bool operator()(int64_t i) const
  {
    return i == 0 || (key[i] >> shift) != (key[i - 1] >> shift);
  }
};

struct StageEmit {
  const int64_t* keyIn;
  int64_t* keyOut;
  int32_t* first;
  PCC_HD void operator()(int64_t rank, int64_t i) const
  {
    keyOut[rank] = keyIn[i];
    first[rank] = int32_t(i);
  }
};

//============================================================================
// step 2: leaves.  Duplicate positions merge into one leaf
// (reduceUnique, RAHT.cpp:108-152).

struct LeafFn {
  Stage L;
  const int32_t* attrs;  // N*A, Morton order
  const int32_t* qpo;    // N*2 or null
  int32_t* dupHf;        // N*A high-pass of duplicates (Haar only) or null
  int A;
  int haar;
  PCC_HD void operator()(int64_t u) const
  {
    int i0 = L.first[u], i1 = L.first[u + 1];
    L.weight[u] = i1 - i0;
    if (L.qpUp) {
      L.qpUp[2 * u] = qpo[2 * size_t(i0)] << 4;
      L.qpUp[2 * u + 1] = qpo[2 * size_t(i0) + 1] << 4;
    }
    for (int k = 0; k < A; k++) {
      uint32_t lf = uint32_t(attrs[size_t(i0) * A + k]);
      for (int i = i0 + 1; i < i1; i++) {
        uint32_t in = uint32_t(attrs[size_t(i) * A + k]);
        if (haar) {
          int32_t d = int32_t(in - lf);
          dupHf[size_t(i) * A + k] = d;
          lf += uint32_t(d >> 1);
        } else {
          lf += in;  // int32 wrap-around like the reference's std::vector<int>
        }
      }
      L.attr[size_t(u) * A + k] = int32_t(lf);
    }
  }
};

//============================================================================
// step 3: one coarser stage from the next finer one.  The three binary
// levels of reduceLevel (RAHT.cpp:157-205) collapse into one merge over the
// <= 8 children of a block, keyed by child slot (x<<2 | y<<1 | z).

struct MergeFn {
  Stage F;  // finer stage (children)
  Stage C;  // coarser stage (parents)
  int A;
  int haar;
  PCC_HD void operator()(int64_t u) const
  {
    int c0 = C.first[u], c1 = C.first[u + 1];
    uint32_t at[8][4];
    int32_t qp[8][2];
    for (int j = 0; j < 8; j++)
      qp[j][0] = qp[j][1] = 0;
    uint32_t present = 0;
    uint32_t wsum = 0;
    for (int c = c0; c < c1; c++) {
      int slot = int((F.key[c] >> F.level) & 7);
      present |= 1u << slot;
      wsum += uint32_t(F.weight[c]);
      for (int k = 0; k < A; k++)
        at[slot][k] = uint32_t(F.attr[size_t(c) * A + k]);
      if (F.qpUp) {
        qp[slot][0] = F.qpUp[2 * c];
        qp[slot][1] = F.qpUp[2 * c + 1];
      }
    }
    C.occ[u] = uint8_t(present);
    C.weight[u] = int32_t(wsum);
    for (int step = 1; step < 8; step <<= 1) {
      for (int lo = 0; lo < 8; lo += 2 * step) {
        int hi = lo + step;
        if (!((present >> hi) & 1))
          continue;
        present &= ~(1u << hi);
        if (!((present >> lo) & 1)) {
          present |= 1u << lo;
          for (int k = 0; k < A; k++)
            at[lo][k] = at[hi][k];
          qp[lo][0] = qp[hi][0];
          qp[lo][1] = qp[hi][1];
          continue;
        }
        for (int k = 0; k < A; k++) {
          if (haar) {
            int32_t d = int32_t(at[hi][k] - at[lo][k]);
            at[lo][k] += uint32_t(d >> 1);
          } else {
            at[lo][k] += at[hi][k];
          }
        }
        qp[lo][0] = (qp[lo][0] + qp[hi][0]) >> 1;
        qp[lo][1] = (qp[lo][1] + qp[hi][1]) >> 1;
      }
    }
    for (int k = 0; k < A; k++)
      C.attr[size_t(u) * A + k] = int32_t(at[0][k]);
    if (C.qpUp) {
      C.qpUp[2 * u] = qp[0][0];
      C.qpUp[2 * u + 1] = qp[0][1];
    }
  }
};

//============================================================================
// the block transform

// RahtKernel coefficients (RAHT.cpp:596-604)
PCC_HD void
raht_ab(int wl, int wr, int64_t& a, int64_t& b)
{
  uint64_t isw = irsqrt64(uint64_t(wl) + uint64_t(wr));
  a = int64_t((uint64_t(isqrt64(uint64_t(wl) << 30)) * isw) >> 40);
  b = int64_t((uint64_t(isqrt64(uint64_t(wr) << 30)) * isw) >> 40);
}

// value * 1/sqrt(w) with the overflow pre-shift of RAHT.cpp:1474-1481
PCC_HD int64_t
scale_rsqrt(int64_t v, int w)
{
  int shift = w > 1024 ? ilog2_u64(uint64_t(w - 1)) >> 1 : 0;
  int64_t rs = int64_t(irsqrt64(uint64_t(w)) >> (40 - shift - kFracBits));
  return fx_mul(v >> shift, rs);
}

// RDOQ: cost in bits of a zero run of length tz (RAHT.cpp:1619-1632)
PCC_TABLE(uint8_t, kZeroRunBins, 11, {1, 2, 3, 5, 5, 7, 7, 9, 9, 11, 11})
PCC_HD int
zero_run_rate(int tz)
{
  if (tz <= 10)
    return kZeroRunBins(tz);
  int a = 32 - clz32(uint32_t(tz - 10));
  return 11 + 2 * a - 1 + 2;
}

// RDOQ classification of a coefficient, 6 bits; eight of them, in scan order,
// make the list a block of the warp kernel publishes (raht_block_warp.cuh):
//   0      all components quantise to zero: never resets the run
//   1      RDOQ removes it whatever the run length: never resets either
//   2      always resets the run (sum |q| >= 3, or RDOQ never fires)
//   3..8   removed if the run before it is at least 1,2,3,5,7,9 long
//   8 + a  removed if the run before it is at least 10 + 2^(a-1), a = 1..30
constexpr int kCodeZero = 0;
constexpr int kCodeRemoved = 1;
constexpr int kCodeHard = 2;

// The smallest zero-run length tz for which the reference's test
// (RAHT.cpp:1617-1636)
//     (Dist2 << 26) < lambda * (Rate(tz) + ((Ratecoeff + 128) >> 8))
// holds, as a code.  Rate(tz) (zero_run_rate) is a non-decreasing step
// function taking 37 values: 1,2,3,5,7,9,11 (tz = 0,1,2,3,5,7,9) and 12 + 2a
// (tz = 10 + 2^(a-1), a = 1..30), so with rc = (Ratecoeff + 128) >> 8 the
// answer is the first of them that is >= floor(lhs / lambda) + 1 - rc.  The
// quotient is below 72 + rc once the test is known to hold for the largest
// rate: a float estimate (invLambda = 1.0f / float(lambda), which depends on
// the quantiser alone and is prepared ahead of the values the block waits
// for) is within one of it, and one 64-bit product settles which.  Dist2 << 26
// wraps like the 64-bit shift it stands for; lambda * (72 + rc) must not
// (lambda is a squared quantiser step times 25 or 35).
PCC_HD int
rdoq_code(int64_t dist2, int64_t lambda, float invLambda, int rateCoeff)
{
  const int64_t lhs = int64_t(uint64_t(dist2) << 26);
  const int rc = (rateCoeff + 128) >> 8;
  if (lhs >= lambda * (72 + rc))
    return kCodeHard;
  if (lhs < lambda)  // (a wrapped, negative left side included)
    return kCodeRemoved;
  int q = int(float(lhs) * invLambda);
  const int64_t prod = lambda * q;
  if (prod > lhs)
    q--;
  else if (prod + lambda <= lhs)
    q++;
  const int need = q + 1 - rc;  // the smallest rate for which the test holds
  // index of the first rate >= need: 0..6 for need <= 11, then rate(i) = 2i
  const int idx = need <= 1 ? 0 : need <= 11 ? int((0x66554433210ull >> (4 * (need - 1))) & 15u)
                                             : need <= 14 ? 7 : (need + 1) >> 1;
  return idx == 0 ? kCodeRemoved : 2 + idx;
}

PCC_TABLE(int16_t, kLutLog, 16,
          {0, 256, 406, 512, 594, 662, 719, 768, 812, 850, 886, 918, 947, 975, 1000, 1024})
PCC_HD int
lut_log(int64_t aq)
{
  return kLutLog(aq < 15 ? int(aq) : 15);
}

// A reconstruction slot that has not been written yet at the current stage
// (the stage's rec array is filled with 0x80 bytes before its blocks run).
// The warp kernel polls the value itself instead of a separate ready flag:
// one L2 round trip per dependency instead of two.
constexpr int64_t kRecNotReady = int64_t(0x8080808080808080ull);

// state words of the zero-run look-back
constexpr int kTzNone = 0;         // nothing published yet
constexpr int kTzTransparent = 1;  // block adds `value` zeros, resets nothing
constexpr int kTzExit = 2;         // `value` is the counter after the block
PCC_HD int tz_pack(int status, int value) { return (value << 2) | status; }
PCC_HD int tz_status(int w) { return w & 3; }
PCC_HD int tz_value(int w) { return w >> 2; }


// tables of findNeighbours / intraDcPred (RAHT.cpp:314-326,375-377,438-440)
PCC_TABLE(uint8_t, kNeighMask, 19,
          {255, 240, 204, 170, 192, 160, 136, 3, 5, 15, 17, 51, 85, 10, 34, 12, 68, 48, 80})
PCC_TABLE(uint8_t, kNeighOffset, 19,
          {0, 35, 21, 14, 49, 42, 28, 1, 2, 3, 4, 5, 6, 10, 12, 17, 20, 33, 34})
PCC_TABLE(uint8_t, kOccuShift, 12, {6, 5, 4, 3, 2, 1, 3, 1, 2, 1, 2, 3})
PCC_HD int neigh_mask(int i) { return kNeighMask(i); }
PCC_HD int neigh_offset(int i) { return kNeighOffset(i); }
PCC_HD int occu_shift(int i) { return kOccuShift(i); }

// index in parent stage P of neighbour i (1..18) of parent p, or -1: the node
// must exist and lie within searchRange entries of p (findNeighbour,
// RAHT.cpp:272-293,342-367)
PCC_HD int
find_parent_neighbour(const Stage& P, int p, int plevel, int64_t cur, int64_t base, int i,
                      int searchRange)
{
  const int64_t np = int64_t(morton3d_add(uint64_t(base), uint64_t(neigh_offset(i))));
  int lo, hi;
  if (np >= cur) {
    lo = p;
    hi = (int64_t(p) + searchRange + 1 < P.n) ? p + searchRange + 1 : P.n;
  } else {
    lo = (p > searchRange) ? p - searchRange : 0;
    hi = p;
  }
  const int end = hi;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if ((P.key[mid] >> plevel) < np)
      lo = mid + 1;
    else
      hi = mid;
  }
  return (lo < end && (P.key[lo] >> plevel) == np) ? lo : -1;
}

// Region qps carried down by the children of one block.  expandLevel
// (RAHT.cpp:210-264) restores weights and sums but never undoes
// reduceLevel's pairwise qp average (RAHT.cpp:187-188): the first child of a
// block inherits the parent's descent value and the first node of each
// right-hand subtree of the block's binary merge tree carries that subtree's
// average.  parentDown == nullptr for the root block (total average).
PCC_HD void
descend_qps(const Stage& S, int c0, int c1, const int32_t* parentDown)
{
  int32_t up[8][2], down[8][2];
  int firstOf[8], child[8];
  uint32_t has = 0;
  for (int j = 0; j < 8; j++) {
    firstOf[j] = j;
    child[j] = -1;
    up[j][0] = up[j][1] = 0;
    down[j][0] = down[j][1] = 0;
  }
  for (int c = c0; c < c1; c++) {
    int slot = int((S.key[c] >> S.level) & 7);
    child[slot] = c;
    has |= 1u << slot;
    up[slot][0] = S.qpUp[2 * c];
    up[slot][1] = S.qpUp[2 * c + 1];
  }
  for (int step = 1; step < 8; step <<= 1)
    for (int lo = 0; lo < 8; lo += 2 * step) {
      int hi = lo + step;
      if (!((has >> hi) & 1))
        continue;
      has &= ~(1u << hi);
      if (!((has >> lo) & 1)) {
        has |= 1u << lo;
        firstOf[lo] = firstOf[hi];
        up[lo][0] = up[hi][0];
        up[lo][1] = up[hi][1];
        continue;
      }
      down[firstOf[hi]][0] = up[hi][0];
      down[firstOf[hi]][1] = up[hi][1];
      up[lo][0] = (up[lo][0] + up[hi][0]) >> 1;
      up[lo][1] = (up[lo][1] + up[hi][1]) >> 1;
    }
  down[firstOf[0]][0] = parentDown ? parentDown[0] : up[0][0];
  down[firstOf[0]][1] = parentDown ? parentDown[1] : up[0][1];
  for (int j = 0; j < 8; j++)
    if (child[j] >= 0) {
      S.qpDown[2 * child[j]] = down[j][0];
      S.qpDown[2 * child[j] + 1] = down[j][1];
    }
}

// zero-run counter after block q-1, i.e. the resolved value of word q
// (decoupled look-back: walk back over transparent blocks to the nearest
// published exit state)
PCC_HD int
tz_lookback(const int* tz, int q)
{
  int acc = 0;
  for (;; q--) {
    int w;
    while (tz_status(w = ld_acquire(&tz[q])) == kTzNone)
      spin_pause();
    if (tz_status(w) == kTzExit)
      return tz_value(w) + acc;
    acc += tz_value(w);
  }
}

struct BlockFn {
  RahtConfig cfg;
  const QpTables* qt;
  Stage S;        // stage being reconstructed (children of the blocks)
  Stage P;        // parent stage; P.n == 0 for the root block
  int32_t* coef;  // planar coefficient buffer, component k at k*coefStride
  int64_t coefStride;
  int64_t coefBase;  // coefficients emitted before this stage
  int qpLayer;
  int acLayer;
  int predInLvl;     // prediction enabled at this stage
  int useFlags;      // ordered dataflow launch: honour done[] / tz[]
  int* tz;           // zero-run look-back words, tz[0] = exit state before
                     // this stage's first block; block p publishes tz[p+1]

  PCC_HD static int slot_of(const Stage& s, int c) { return int((s.key[c] >> s.level) & 7); }

  PCC_HD void wait_done(int q) const
  {
    if (!useFlags)
      return;
    while (!ld_acquire(&P.done[q]))
      spin_pause();
  }

  PCC_HD int lookback(int p) const { return tz_lookback(tz, p); }

  PCC_HD void operator()(int64_t pb) const
  {
    const int p = int(pb);
    const int A = cfg.A;
    const bool root = P.n == 0;
    const int c0 = root ? 0 : P.first[p];
    const int c1 = root ? S.n : P.first[p + 1];

    int64_t buf[6][8];
    int w[32];
    int nodeQp[8][2];
    int child[8];
    for (int j = 0; j < 8; j++) {
      w[j] = 0;
      child[j] = -1;
      nodeQp[j][0] = nodeQp[j][1] = 0;
      for (int k = 0; k < 6; k++)
        buf[k][j] = 0;
    }
    int64_t(*pred)[8] = &buf[A];
    uint32_t occ = 0;

    for (int c = c0; c < c1; c++) {
      int slot = slot_of(S, c);
      child[slot] = c;
      w[slot] = S.weight[c];
      occ |= 1u << slot;
      if (cfg.isEncoder)
        for (int k = 0; k < A; k++)
          buf[k][slot] = fx_from_int(S.attr[size_t(c) * A + k]);
    }
    const int nodeCnt = cfg.ext ? c1 - c0 : 0;

    //-- region qps carried down (written by PrepFn for non-root stages)
    if (cfg.hasQp) {
      if (root)
        descend_qps(S, c0, c1, nullptr);
      for (int j = 0; j < 8; j++)
        if (child[j] >= 0) {
          nodeQp[j][0] = S.qpDown[2 * child[j]] >> 4;
          nodeQp[j][1] = S.qpDown[2 * child[j] + 1] >> 4;
        }
    }

    //-- weight tree (mkWeightTree, RAHT.cpp:742-771)
    for (int g = 0; g < 3; g++)
      for (int i = 0; i < 4; i++) {
        int l = w[8 * g + 2 * i], r = w[8 * g + 2 * i + 1];
        w[8 * g + 8 + i] = l + r;
        w[8 * g + 12 + i] = (l && r) ? l + r : 0;
      }

    //-- neighbour search and prediction gating (RAHT.cpp:1391-1432, 299-416)
    bool enablePred = predInLvl != 0;
    int count = root ? 19 : 0;
    int pidx[19];
    if (predInLvl) {
      if (cfg.ext && nodeCnt == 1) {
        enablePred = false;
        count = 19;
      } else if (P.nn[p] < cfg.thr0) {
        enablePred = false;
      } else {
        const int plevel = S.level + 3;
        const int64_t cur = P.key[p] >> plevel;
        const int64_t base = int64_t(morton3d_add(uint64_t(cur), ~uint64_t(0)));
        pidx[0] = p;
        count = 1;
        for (int i = 1; i < 19; i++) {
          pidx[i] = -1;
          if (!(occ & neigh_mask(i)))
            continue;
          pidx[i] = find_parent_neighbour(P, p, plevel, cur, base, i, cfg.searchRange);
          count += pidx[i] >= 0;
        }
        if (count < cfg.thr1)
          enablePred = false;
      }
    }
    if (root || predInLvl)
      for (int c = c0; c < c1; c++)
        S.nn[c] = count;

    //-- encoder: normalise and transform the sums (independent of any other
    //   block, so done before waiting on neighbours)
    if (cfg.isEncoder) {
      if (!cfg.haar)
        for (int j = 0; j < 8; j++)
          if (w[j] > 1)
            for (int k = 0; k < A; k++)
              buf[k][j] = scale_rsqrt(buf[k][j], w[j]);
      transform(A, buf, w, true);
    }

    //-- prediction (intraDcPred, RAHT.cpp:421-589)
    if (enablePred) {
      const uint8_t kMasks[19] = {255, 240, 204, 170, 192, 160, 136, 3, 5, 15,
                                  17,  51,  85,  10,  34,  12,  68,  48, 80};
      const uint8_t kShift[12] = {6, 5, 4, 3, 2, 1, 3, 1, 2, 1, 2, 3};
      int wsum[8];
      for (int j = 0; j < 8; j++)
        wsum[j] = -1;
      int64_t limLow = 0, limHigh = 0;
      const int64_t fracMul = cfg.ext ? 1 : (int64_t(1) << kFracBits);
      const int parentOnly = cfg.subnode ? 7 : 19;
      for (int i = 0; i < 19; i++) {
        int q = pidx[i];
        if (q < 0)
          continue;
        int64_t v[3];
        for (int k = 0; k < A; k++)
          v[k] = P.rec[size_t(q) * A + k];
        if (i) {
          if (10 * v[0] <= limLow || 10 * v[0] >= limHigh)
            continue;
        } else {
          limLow = 2 * v[0];
          limHigh = 25 * v[0];
        }
        const int wp = cfg.predWeightParent[i];
        for (int k = 0; k < A; k++)
          v[k] *= wp * fracMul;
        uint32_t mask = kMasks[i] & occ;
        uint32_t cmask = 0;  // slots served by an already reconstructed child
        int sh = 0, sgn = 1;
        uint32_t nocc = 0;
        int cfirst = 0;
        if (i >= parentOnly && q < p) {
          // neighbour block precedes us in Morton order: its children are
          // (or will shortly be) reconstructed at this stage
          const int ii = i - 7;
          sh = kShift[ii];
          sgn = ii < 9 ? 1 : -1;
          nocc = P.occ[q];
          cmask = (ii < 9 ? (nocc >> sh) : (nocc << sh)) & mask & 0xff;
          if (cmask) {
            cfirst = P.first[q];
            wait_done(q);
          }
        }
        const int wc = i >= 7 ? cfg.predWeightChild[i - 7] : 0;
        for (int j = 0; j < 8; j++) {
          if (!((mask >> j) & 1))
            continue;
          if ((cmask >> j) & 1) {
            int nslot = j + sgn * sh;
            int c = cfirst + popc32(nocc & ((1u << nslot) - 1));
            wsum[j] += wc;
            for (int k = 0; k < A; k++)
              pred[k][j] += S.rec[size_t(c) * A + k] * (wc * fracMul);
          } else {
            wsum[j] += wp;
            for (int k = 0; k < A; k++)
              pred[k][j] += v[k];
          }
        }
      }
      for (int j = 0; j < 8; j++) {
        if (!((occ >> j) & 1))
          continue;
        int d = wsum[j] + 1;
        int64_t div = (32768 + d / 2) / d;  // == kDivisors[wsum], RAHT.cpp:445-451
        for (int k = 0; k < A; k++) {
          int64_t v = fx_mul(pred[k][j], div);
          if (cfg.haar)
            v = (v >> kFracBits) << kFracBits;
          else if (w[j] > 1)
            v = fx_mul(v, int64_t(isqrt64(uint64_t(w[j]) << (2 * kFracBits))));
          pred[k][j] = v;
        }
      }
      transform(A, pred, w, true);
    }

    //-- coefficients in scan order (RAHT.cpp:1558-1724)
    const int kScan[8] = {0, 4, 2, 1, 6, 5, 3, 7};
    LayerQp lq;
    lq.luma = qt->layers[qpLayer][0];
    lq.chromaOffset = qt->layers[qpLayer][1];
    lq.maxQp = cfg.maxQp;
    lq.fixedPointQpOffset = cfg.fixedPointQpOffset;

    const bool rdoq = cfg.isEncoder && !cfg.haar;
    int kind[8];         // per scanned coefficient: 0 zero, 1 soft, 2 hard
    int64_t dist2[8];
    int rateCoeff[8];
    int64_t lambda[8];
    int ncoef = 0;
    bool anySoft = false, anyHard = false;
    if (cfg.isEncoder) {
      for (int si = 0; si < 8; si++) {
        int idx = kScan[si];
        if ((si && !w[24 + idx]) || (!root && !idx))
          continue;
        if (enablePred)
          for (int k = 0; k < A; k++)
            buf[k][idx] -= pred[k][idx];
        if (rdoq) {
          Quantizer q[2];
          make_quantizers(lq, nodeQp[idx][0], nodeQp[idx][1], q);
          int64_t sum = 0, d2 = 0;
          int rc = 0;
          for (int k = 0; k < A; k++) {
            int64_t c = fx_round(buf[k][idx]);
            d2 += c * c;
            int64_t qc = q[k < 1 ? k : 1].quantize(c << kAttrShift);
            int64_t aq = qc < 0 ? -qc : qc;
            sum += aq;
            rc += lut_log(aq);
          }
          int64_t l0 = q[0].scale(1);
          kind[ncoef] = sum == 0 ? 0 : (sum < 3 ? 1 : 2);
          anySoft |= kind[ncoef] == 1;
          anyHard |= kind[ncoef] == 2;
          dist2[ncoef] = d2;
          rateCoeff[ncoef] = rc;
          lambda[ncoef] = l0 * l0 * (A == 1 ? 25 : 35);
        }
        ncoef++;
      }
    }

    // zero-run counter protocol (decoupled look-back).  Word tz[p + 1] is the
    // state after block p; tz[0] the state before the stage's first block.
    //  * a block whose coefficients all quantise to zero is transparent: it
    //    adds ncoef to whatever counter it is handed;
    //  * a block holding a coefficient that resets the counter
    //    unconditionally knows its exit state without knowing its entry state;
    //  * the entry state is needed only if a coefficient whose RDOQ decision
    //    matters precedes the block's first unconditional reset.
    bool flag[8];
    for (int i = 0; i < 8; i++)
      flag[i] = false;
    bool published = false;
    if (rdoq) {
      // with AC-coefficient qp offsets the final quantiser differs from the
      // one the RDOQ test uses, so the decision matters even for kind 0
      const bool zeroMatters = cfg.numAcLayers > 0;
      int firstSensitive = -1, firstHard = -1, lastHard = -1;
      for (int i = 0; i < ncoef; i++) {
        if ((kind[i] == 1 || (kind[i] == 0 && zeroMatters)) && firstSensitive < 0)
          firstSensitive = i;
        if (kind[i] == 2) {
          if (firstHard < 0)
            firstHard = i;
          lastHard = i;
        }
      }
      if (useFlags && !anySoft && !anyHard)
        st_release(&tz[p + 1], tz_pack(kTzTransparent, ncoef));
      if (useFlags && anyHard) {
        // every decision after the last hard reset is local
        int t = 0;
        for (int i = lastHard + 1; i < ncoef; i++)
          t = step_tz(t, kind[i], dist2[i], lambda[i], rateCoeff[i], nullptr);
        st_release(&tz[p + 1], tz_pack(kTzExit, t));
        published = true;
      }
      const bool needEntry =
        firstSensitive >= 0 && (firstHard < 0 || firstSensitive < firstHard);
      int t = 0;
      if (!useFlags)
        t = tz_value(tz[p]);  // in-order execution: previous block's exit
      else if (needEntry)
        t = lookback(p);
      for (int i = 0; i < ncoef; i++)
        t = step_tz(t, kind[i], dist2[i], lambda[i], rateCoeff[i], &flag[i]);
      if (!useFlags) {
        tz[p + 1] = tz_pack(kTzExit, t);
        published = true;
      } else if (!published && needEntry) {
        // the entry state has just been resolved, so the exit state is known
        st_release(&tz[p + 1], tz_pack(kTzExit, t));
        published = true;
      }
    }

    // quantise / dequantise (RAHT.cpp:1672-1723)
    {
      int64_t pos = coefBase + c0 - (root ? 0 : p);
      int ci = 0;
      for (int si = 0; si < 8; si++) {
        int idx = kScan[si];
        if ((si && !w[24 + idx]) || (!root && !idx))
          continue;
        int off0 = nodeQp[idx][0], off1 = nodeQp[idx][1];
        if (idx && acLayer < cfg.numAcLayers) {
          off0 += qt->acQps[acLayer][idx - 1][0];
          off1 += qt->acQps[acLayer][idx - 1][1];
        }
        Quantizer q[2];
        make_quantizers(lq, off0, off1, q);
        for (int k = 0; k < A; k++) {
          const Quantizer& qk = q[k < 1 ? k : 1];
          int64_t qc;
          if (cfg.isEncoder) {
            int64_t c = flag[ci] ? 0 : fx_round(buf[k][idx]);
            qc = qk.quantize(c << kAttrShift);
            coef[k * coefStride + pos] = int32_t(qc);
          } else {
            qc = coef[k * coefStride + pos];
          }
          pred[k][idx] +=
            fx_from_int(div_exp2_round_half_up(qk.scale(qc), kAttrShift));
        }
        pos++;
        ci++;
      }
    }

    //-- DC from the parent's un-scaled reconstruction (RAHT.cpp:1726-1742)
    if (!root)
      for (int k = 0; k < A; k++) {
        int64_t v = P.recUs[size_t(p) * A + k];
        pred[k][0] = cfg.ext ? v : v * (int64_t(1) << (kFracBits - 2));
      }

    transform(A, pred, w, false);

    //-- store reconstructions (RAHT.cpp:1754-1806)
    for (int j = 0; j < 8; j++) {
      int c = child[j];
      if (c < 0)
        continue;
      for (int k = 0; k < A; k++) {
        int64_t v = pred[k][j];
        S.recUs[size_t(c) * A + k] = cfg.ext ? v : fx_round(v * 4);
        if (!cfg.haar && w[j] > 1)
          v = scale_rsqrt(v, w[j]);
        S.rec[size_t(c) * A + k] = cfg.ext ? v : fx_round(v);
      }
    }
    if (useFlags && !root) {
#if defined(__CUDA_ARCH__)
      __threadfence();
#endif
      st_release(&P.done[p], 1);
      // transparent blocks still close their look-back chain so that later
      // blocks never walk further than to their immediate neighbourhood
      if (rdoq && !published)
        st_release(&tz[p + 1], tz_pack(kTzExit, lookback(p) + ncoef));
    }
  }

  // one step of the zero-run counter (RAHT.cpp:1617-1662)
  PCC_HD static int step_tz(int t, int kind, int64_t dist2, int64_t lambda,
                            int rateCoeff, bool* flag)
  {
    bool f = false;
    if (kind < 2) {
      int rate = zero_run_rate(t) + ((rateCoeff + 128) >> 8);
      f = (dist2 << 26) < lambda * rate;
    }
    if (flag)
      *flag = f;
    return (f || kind == 0) ? t + 1 : 0;
  }

  // fwdTransformBlock222 / invTransformBlock222 (RAHT.cpp:671-737)
  PCC_HD void transform(int nbuf, int64_t b[][8], const int* w, bool fwd) const
  {
    const int kA[12] = {0, 2, 4, 6, 0, 4, 1, 5, 0, 1, 2, 3};
    const int kB[12] = {1, 3, 5, 7, 2, 6, 3, 7, 4, 5, 6, 7};
    for (int n = 0; n < 12; n++) {
      int i = fwd ? n : 11 - n;
      int i0 = kA[i], i1 = kB[i];
      int wl = w[2 * i], wr = w[2 * i + 1];
      if (wl + wr == 0)
        continue;
      if (!wl || !wr) {
        if (!wl)
          for (int k = 0; k < nbuf; k++) {
            int64_t t = b[k][i0];
            b[k][i0] = b[k][i1];
            b[k][i1] = t;
          }
        continue;
      }
      if (cfg.haar) {
        for (int k = 0; k < nbuf; k++) {
          if (fwd) {
            int64_t hf = b[k][i1] - b[k][i0];
            b[k][i0] += (hf >> (1 + kFracBits)) << kFracBits;
            b[k][i1] = hf;
          } else {
            int64_t hf = b[k][i1];
            int64_t l = b[k][i0] - ((hf >> (1 + kFracBits)) << kFracBits);
            b[k][i0] = l;
            b[k][i1] = hf + l;
          }
        }
        continue;
      }
      int64_t ca, cb;
      raht_ab(wl, wr, ca, cb);
      for (int k = 0; k < nbuf; k++) {
        int64_t x0 = b[k][i0], x1 = b[k][i1];
        if (fwd) {
          b[k][i0] = fx_mul(x1, cb) + fx_mul(ca, x0);
          b[k][i1] = fx_mul(x1, ca) - fx_mul(cb, x0);
        } else {
          b[k][i0] = fx_mul(x0, ca) - fx_mul(cb, x1);
          b[k][i1] = fx_mul(x0, cb) + fx_mul(ca, x1);
        }
      }
    }
  }
};


//============================================================================
// Work of a stage that needs no other block of the same stage, one thread
// per block: the qp descent, and the complete treatment of blocks with a
// single child.  Such a block has no coefficients (its DC is inherited,
// RAHT.cpp:1727-1742, and there is no AC), so its reconstruction is the
// parent's value passed through; with rahtExtension it is also never
// predicted (RAHT.cpp:1399-1401).  Chains of single-child levels dominate
// sparse (LiDAR) clouds; taking them out leaves the ordered dataflow kernel
// with the blocks that really transform.

struct PrepFn {
  RahtConfig cfg;
  Stage S;
  Stage P;
  int predInLvl;
  int* tzByBlock;  // block-indexed look-back words (or null): a single-child
                   // block publishes "transparent, 0 coefficients"
  int mode = 0;    // 0: everything; 1: the value-free part only (qps, neighbour
                   // counts); 2: the values only (pass-through)
  PCC_HD void operator()(int64_t pb) const
  {
    const int p = int(pb);
    const int c0 = P.first[p], c1 = P.first[p + 1];
    if (cfg.hasQp && mode != 2)
      descend_qps(S, c0, c1, &P.qpDown[2 * p]);
    if (c1 - c0 != 1)
      return;
    const int c = c0;
    const int A = cfg.A;
    if (predInLvl && mode != 2) {
      int count = 0;
      if (cfg.ext) {
        count = 19;
      } else if (P.nn[p] >= cfg.thr0) {
        const int plevel = S.level + 3;
        const int64_t cur = P.key[p] >> plevel;
        const int64_t base = int64_t(morton3d_add(uint64_t(cur), ~uint64_t(0)));
        const int occ = P.occ[p];
        count = 1;
        for (int i = 1; i < 19; i++)
          if (occ & neigh_mask(i))
            count += find_parent_neighbour(P, p, plevel, cur, base, i, cfg.searchRange) >= 0;
      }
      S.nn[c] = count;
    }
    if (mode == 1)
      return;
    const int wgt = S.weight[c];
    for (int k = 0; k < A; k++) {
      int64_t v = P.recUs[size_t(p) * A + k];
      int64_t x = cfg.ext ? v : v * (int64_t(1) << (kFracBits - 2));
      S.recUs[size_t(c) * A + k] = cfg.ext ? x : fx_round(x * 4);
      if (!cfg.haar && wgt > 1)
        x = scale_rsqrt(x, wgt);
      S.rec[size_t(c) * A + k] = cfg.ext ? x : fx_round(x);
    }
    P.done[p] = 1;
    if (tzByBlock)
      tzByBlock[p + 1] = tz_pack(kTzTransparent, 0);
  }
};

// blocks that the ordered kernel has to run
struct MultiChildPred {
  const int32_t* first;
  PCC_HD bool operator()(int64_t p) const { return first[p + 1] - first[p] >= 2; }
};
struct WorklistEmit {
  int32_t* list;
  PCC_HD void operator()(int64_t rank, int64_t p) const { list[rank] = int32_t(p); }
};

// run fn(p) only for blocks with at least two children (thread-per-block path)
template<class Fn>
struct SkipSinglesFn {
  Fn fn;
  PCC_HD void operator()(int64_t p) const
  {
    if (fn.P.first[p + 1] - fn.P.first[p] >= 2)
      fn(p);
  }
};

// hand the zero-run counter to the next stage: dst[0] = exit state after the
// last of n blocks (n from device memory when countPtr != null)
struct TzCarryFn {
  const int* tzSrc;
  const int* countPtr;
  int hostCount;
  int* tzDst;
  PCC_HD void operator()(int64_t) const
  {
    int n = countPtr ? *countPtr : hostCount;
    tzDst[0] = tz_pack(kTzExit, tz_lookback(tzSrc, n));
  }
};

//============================================================================
// last step: duplicate points (RAHT.cpp:1840-1964) and write-back
// (RAHT.cpp:1967-1975), one thread per leaf.

// the part of an attribute the tail needs (see AttrSet in raht_block_warp.cuh)
struct TailSet {
  int A, base;
  int maxQp, fixedPointQpOffset;
  int qpLayer;
  const QpTables* qt;
  int32_t* coef;
  int64_t coefStride;
};

struct TailFn {
  RahtConfig cfg;          // cfg.A: components of all sets together
  int numSets;
  TailSet set[2];
  Stage L;
  const int32_t* attrsIn;  // N*A source values (encoder), Morton order
  const int32_t* dupHf;    // Haar high-pass of the duplicates, or null
  int32_t* attrsOut;       // N*A
  int64_t coefBase;        // coefficients emitted by the stages
  int hasStages;           // 0 when all points share one position

  PCC_HD void operator()(int64_t ub) const
  {
    const int u = int(ub);
    const int A = cfg.A;
    const int i0 = L.first[u];
    const int wt = L.first[u + 1] - i0;
    auto finish = [&](int64_t v) -> int32_t {
      return cfg.ext ? int32_t((v + kOneHalf) >> kFracBits) : int32_t(v);
    };
    if (wt == 1) {
      for (int k = 0; k < A; k++)
        attrsOut[size_t(i0) * A + k] =
          finish(hasStages ? L.rec[size_t(u) * A + k] : 0);
      return;
    }
    int off0 = 0, off1 = 0;
    if (cfg.hasQp) {
      const int32_t* src = hasStages ? L.qpDown : L.qpUp;
      off0 = src[2 * u] >> 4;
      off1 = src[2 * u + 1] >> 4;
    }
    const int64_t sq = int64_t(isqrt64(uint64_t(wt) << (2 * kFracBits)));
    const int64_t pos0 = coefBase + (i0 - u);
    for (int si = 0; si < numSets; si++) {
      const TailSet& ts = set[si];
      LayerQp lq;
      lq.luma = ts.qt->layers[ts.qpLayer][0];
      lq.chromaOffset = ts.qt->layers[ts.qpLayer][1];
      lq.maxQp = ts.maxQp;
      lq.fixedPointQpOffset = ts.fixedPointQpOffset;
      Quantizer q[2];
      make_quantizers(lq, off0, off1, q);
      for (int kk = 0; kk < ts.A; kk++) {
        const int k = ts.base + kk;
        const Quantizer& qk = q[kk < 1 ? kk : 1];
        int64_t attrSum = fx_from_int(L.attr[size_t(u) * A + k]);
        int64_t r = hasStages ? L.rec[size_t(u) * A + k] : 0;
        int64_t recDc = cfg.ext ? r : fx_from_int(r);
        if (!cfg.haar)
          recDc = fx_mul(recDc, sq);
        for (int w = wt - 1; w > 0; w--) {
          int64_t ca, cb;
          raht_ab(w, 1, ca, cb);
          int64_t pos = pos0 + (wt - 1 - w);
          int64_t qc;
          if (cfg.isEncoder) {
            int64_t t0, t1;
            if (cfg.haar) {
              // undo the lifting step; the high-pass (right - left) is the
              // stored difference itself
              t1 = fx_from_int(dupHf[size_t(i0 + w) * A + k]);
              attrSum -= t1 >> 1;
            } else {
              t1 = fx_from_int(attrsIn[size_t(i0 + w) * A + k]);
              attrSum -= t1;
              t0 = scale_rsqrt(attrSum, w);
              t1 = fx_mul(t1, ca) - fx_mul(cb, t0);
            }
            qc = qk.quantize(fx_round(t1) << kAttrShift);
            ts.coef[kk * ts.coefStride + pos] = int32_t(qc);
          } else {
            qc = ts.coef[kk * ts.coefStride + pos];
          }
          int64_t hf = fx_from_int(div_exp2_round_half_up(qk.scale(qc), kAttrShift));
          int64_t left, right;
          if (cfg.haar) {
            left = recDc - ((hf >> (1 + kFracBits)) << kFracBits);
            right = hf + left;
          } else {
            left = fx_mul(recDc, ca) - fx_mul(cb, hf);
            right = fx_mul(recDc, cb) + fx_mul(ca, hf);
          }
          recDc = left;
          attrsOut[size_t(i0 + w) * A + k] = finish(cfg.ext ? right : fx_round(right));
          if (w == 1)
            attrsOut[size_t(i0) * A + k] = finish(cfg.ext ? left : fx_round(left));
        }
      }
    }
  }
};

// single point (RAHT.cpp:998-1017)
struct SinglePointFn {
  RahtConfig cfg;
  const QpTables* qt;
  const int32_t* qpo;
  int32_t* attrs;
  int32_t* coef;
  int64_t coefStride;
  PCC_HD void operator()(int64_t) const
  {
    LayerQp lq;
    lq.luma = qt->layers[0][0];
    lq.chromaOffset = qt->layers[0][1];
    lq.maxQp = cfg.maxQp;
    lq.fixedPointQpOffset = cfg.fixedPointQpOffset;
    Quantizer q[2];
    make_quantizers(lq, qpo ? qpo[0] : 0, qpo ? qpo[1] : 0, q);
    for (int k = 0; k < cfg.A; k++) {
      const Quantizer& qk = q[k < 1 ? k : 1];
      int64_t c;
      if (cfg.isEncoder) {
        c = qk.quantize(int64_t(attrs[k]) << kAttrShift);
        coef[k * coefStride] = int32_t(c);
      } else {
        c = coef[k * coefStride];
      }
      attrs[k] = int32_t(div_exp2_round_half_up(qk.scale(c), kAttrShift));
    }
  }
};

}  // namespace pccb200
