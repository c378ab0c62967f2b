// raht_block_warp.cuh — the top-down block transform as a warp-cooperative
// dataflow kernel (device only).  Same arithmetic, statement for statement, as
// BlockFn in raht_core.cuh (which stays the host-testable definition); what
// changes is the mapping onto the machine:
//
//   * one warp per block of siblings; lane = component * 8 + child slot, so
//     the 2x2x2 block of a colour attribute fills 24 lanes and the three
//     butterfly stages are __shfl_xor exchanges with lanes 1, 2 and 4 away;
//     the 18 neighbour look-ups are binary searches run by 18 lanes at once
//     (k_block_geom), and lane i < 19 fetches neighbour i's data;
//   * everything lives in registers (no per-thread arrays in local memory);
//   * warps claim blocks in Morton order through a global ticket, one block
//     at a time, so every lower-numbered block is owned by a running warp: a
//     warp may wait for the reconstruction slot of any earlier block
//     (sub-node prediction) and for its zero-run classification (RDOQ)
//     without any risk of deadlock, whatever the residency;
//   * blocks with a single child never reach this kernel (PrepFn).
//
// Reference: the block loop of uraht_process, tmc3/RAHT.cpp:1306-1808.
#pragma once

#include "raht_core.cuh"

namespace pccb200 {

// One attribute of the pass.  Attributes coded on the same positions share
// everything that follows from geometry (tree, worklists, neighbour tables,
// weights, butterfly constants, the dependency chain); each keeps its own
// quantisers, prediction range test, coefficient planes and zero-run stream.
// Component rows of the warp (lane >> 3): [base, base + A).
struct AttrSet {
  int A;     // components (1..3)
  int base;  // first component row
  int maxQp, fixedPointQpOffset, numAcLayers;
  int qpLayer, acLayer;  // of the current stage
  const QpTables* qt;
  int32_t* coef;         // planar coefficients, component kk at kk * coefStride
  int64_t coefStride;
  const struct TzRegion* regions;  // zero-run state words of every stage so far
  unsigned long long* state;       // regions[stageIdx].state (kernel parameter: no load on
                                   //   the critical path)
};

constexpr int kMaxSets = 2;

struct WarpBlockArgs {
  RahtConfig cfg;     // cfg.A = components of all sets together (<= 4)
  int numSets;
  AttrSet set[kMaxSets];
  Stage S;
  Stage P;            // P.n == 0: root block
  int64_t coefBase;
  int predInLvl;
  const int32_t* worklist;  // block indices in Morton order (null for the root)
  int32_t* geom;            // kGeomStride ints per worklist entry (see k_block_geom)
  const int* count;         // number of worklist entries (device memory)
  int64_t ab11a, ab11b;     // RahtKernel(1, 1), the commonest butterfly
  int stageIdx;             // index of this stage in the sets' regions (0 = root)
  int pollNs;               // sleep between polls of a value still being produced
  // wavefront schedule (raht_wave.cuh): ticket i runs the block of row
  // order[i] (worklist rank + orderBase), rows sorted by dependency level
  const int32_t* order;
  int orderBase;
};

// Zero-run bookkeeping of one stage, indexed by worklist rank t: state[t + 1]
// is block t's 64-bit state word (zero = nothing published yet):
//   bits 1:0   status (kTzTransparent / kTzExit / kTzClassified)
//   bits 5:2   value: the block's coefficient count (transparent, classified)
//              or the run length after the block (exit); at most 8
//   bits 53:6  classification of its coefficients in scan order, 6 bits each
//              (see below; present with every status once the block has soft
//              coefficients)
// One word, written with one relaxed 64-bit store: a consumer needs no second
// load and the producer no release fence (the fence of a store-release waits
// for the block's earlier stores to reach L2 -- on the critical path of the
// chain, twice per block).
struct TzRegion {
  unsigned long long* state;
  const int* count;
};

__device__ __forceinline__ unsigned long long
state_pack(int status, int value, unsigned long long codes)
{
  return (unsigned long long)(status | (value << 2)) | codes << 6;
}
__device__ __forceinline__ unsigned long long
ld_state(const unsigned long long* p)
{
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void
st_state(unsigned long long* p, unsigned long long v)
{
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

constexpr int kTzClassified = 3;  // word status: list published, outcome pending

// Developer build (make EXTRA=-DPCCB200_HOP_STATS; tools/hop_profile.py): where
// the cycles of a block go, summed per descent step over all units, by lane 0
// with clock64() and atomicAdd.  The default build contains none of it.
#ifdef PCCB200_HOP_STATS
enum HopCounter {
  kHopBlocks,          // blocks processed
  kHopChildPolls,      // sleeps in the child-value poll
  kHopChildCycles,     // cycles in the child-value poll (first load to last arrival)
  kHopClassifyCycles,  // last child value -> the block's first state word
  kHopTzCalls,         // look-backs
  kHopTzPolls,         // sleeps inside look-backs
  kHopTzCycles,        // cycles inside look-backs
  kHopTailCycles,      // last look-back (or the state word) -> st_rec issued
  kHopExtraLoads,      // ld_state issued by look-backs beyond the two prefetched words
  kHopWalk1,           // look-backs that read 1, 2, 3-4, 5-8, more than 8 words
  kHopWalk2,
  kHopWalk4,
  kHopWalk8,
  kHopWalkMore,
  kHopCounters
};
constexpr int kHopStages = 32;
__device__ unsigned long long g_hopStats[kHopStages][kHopCounters];
__device__ __forceinline__ void
hop_add(int stage, int c, long long v)
{
  if ((threadIdx.x & 31) == 0)
    atomicAdd(&g_hopStats[stage][c], (unsigned long long)v);
}
#  define HOP_ONLY(...) __VA_ARGS__
#else
#  define HOP_ONLY(...)
#endif
#define HOP_STAT(c, v) HOP_ONLY(hop_add(a.stageIdx, c, v);)
#define HOP_CLOCK(x) HOP_ONLY(x = clock64();)

constexpr int kWarpBlockThreads = 256;
#ifndef PCCB200_BLOCK_MIN_CTAS
#  define PCCB200_BLOCK_MIN_CTAS 3  // resident CTAs per SM the block kernel is compiled for
#endif
constexpr int kGeomStride = 20;     // ints per block: 19 neighbour indices + count

__device__ __forceinline__ int64_t
shfl_xor_i64(int64_t v, int m)
{
  return (int64_t)__shfl_xor_sync(0xffffffffu, (long long)v, m);
}
__device__ __forceinline__ int64_t
shfl_i64(int64_t v, int src)
{
  return (int64_t)__shfl_sync(0xffffffffu, (long long)v, src);
}

// RahtKernel(wl, wr) out of line: the three butterfly levels share one copy of
// the (long) square-root arithmetic, which keeps the kernel's hot code small
// (instruction-cache misses showed up as a top stall reason on the big stages)
struct RahtAB {
  int64_t a, b;
};
#ifdef PCCB200_INLINE_AB
__device__ __forceinline__ RahtAB
#else
__device__ __noinline__ RahtAB
#endif
raht_ab_shared(int wl, int wr)
{
  RahtAB r;
  raht_ab(wl, wr, r.a, r.b);
  return r;
}

// one butterfly stage; every lane calls it (the shuffle is unconditional)
struct Bfly {
  int64_t a, b;
  bool both, swap, lo;
};

__device__ __forceinline__ int64_t
bfly_fwd(int64_t x, const Bfly& f, int dist, bool haar)
{
  const int64_t y = shfl_xor_i64(x, dist);
  if (f.both) {
    if (haar) {
      // lo holds left, hi holds right; hf = right - left
      if (f.lo) {
        int64_t hf = y - x;
        return x + ((hf >> (1 + kFracBits)) << kFracBits);
      }
      return x - y;
    }
    return f.lo ? fx_mul(y, f.b) + fx_mul(f.a, x) : fx_mul(x, f.a) - fx_mul(f.b, y);
  }
  return f.swap ? y : x;
}

__device__ __forceinline__ int64_t
bfly_inv(int64_t x, const Bfly& f, int dist, bool haar)
{
  const int64_t y = shfl_xor_i64(x, dist);
  if (f.both) {
    if (haar) {
      if (f.lo)  // x = lf, y = hf
        return x - ((y >> (1 + kFracBits)) << kFracBits);
      // x = hf, y = lf
      return x + (y - ((x >> (1 + kFracBits)) << kFracBits));
    }
    return f.lo ? fx_mul(x, f.a) - fx_mul(f.b, y) : fx_mul(y, f.b) + fx_mul(f.a, x);
  }
  return f.swap ? y : x;
}

// reconstruction values are exchanged between blocks through L2: relaxed
// 64-bit accesses, the value itself says whether it has been produced
__device__ __forceinline__ int64_t
ld_rec(const int64_t* p)
{
  long long v;
  asm volatile("ld.relaxed.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return int64_t(v);
}
__device__ __forceinline__ void
st_rec(int64_t* p, int64_t v)
{
  asm volatile("st.relaxed.gpu.global.s64 [%0], %1;" ::"l"(p), "l"((long long)v) : "memory");
}
__device__ __forceinline__ int64_t
poll_rec(const int64_t* p)
{
  int64_t v = ld_rec(p);
  while (v == kRecNotReady) {
    __nanosleep(32);
    v = ld_rec(p);
  }
  return v;
}

// run-length threshold of a classification code (kCode*, raht_core.cuh)
__device__ __forceinline__ int
thr_decode(int code)  // code >= 3
{
  return code < 9 ? int((0x975321u >> (4 * (code - 3))) & 15u) : 10 + (1 << (code - 9));
}

// Is the run of non-resetting coefficients that ends just before block t of
// stage a.stageIdx at least `need` long?  Walks back over the published
// classification of earlier blocks (this stage, then earlier stages); waits
// only for blocks that have not classified their coefficients yet, never for
// another block's own answer (whatever a block publishes later is consistent
// with its list, so the answer does not depend on when a word is read).
//
// Every lane walks the stream of its own attribute (the lanes of an
// attribute read the same words and agree; the attributes of a pass walk side
// by side in the same instruction stream).  Two warp-cooperative variants --
// 32 predecessors fetched per round trip, and two streams at once with the
// first batch fetched when the block starts -- were measured slower on the
// textured frame: what bounds a stage there is
// not the memory latency of the walk but the instruction issue the waiting
// warps take from the one warp that can make progress, and a heavier loop
// around the poll makes every waiting warp more expensive.
__device__ __forceinline__ bool
tz_run_at_least(const AttrSet& st, const int stageIdx, const int pollNs, int t, int need,
                const unsigned long long wPre1, const unsigned long long wPre2)
{
  if (need <= 0)
    return true;
  int req = need;  // positions 1..req behind the block must not reset the run
  int acc = 0;     // positions already verified
  int s = stageIdx;
  const unsigned long long* state = st.state;
  int u = t - 1;
  HOP_ONLY(int hopWords = 0; int hopLoads = 0; int hopSleeps = 0;)
  HOP_ONLY(auto hop_done = [&]() {
    hop_add(stageIdx, hopWords <= 1 ? kHopWalk1 : hopWords == 2 ? kHopWalk2 : hopWords <= 4 ? kHopWalk4
            : hopWords <= 8 ? kHopWalk8 : kHopWalkMore, 1);
    hop_add(stageIdx, kHopExtraLoads, hopLoads);
    hop_add(stageIdx, kHopTzPolls, hopSleeps);
  };)
  for (;;) {
    if (u < 0) {
      if (--s < 0) {
        HOP_ONLY(hop_done();)
        return acc >= req;  // start of the call: the counter starts at 0
      }
      const TzRegion rg = st.regions[s];
      state = rg.state;
      u = *rg.count - 1;
      continue;
    }
    // (words fetched ahead are as good as fresh ones unless they were empty)
    unsigned long long w =
      (s == stageIdx && u == t - 1) ? wPre1 : (s == stageIdx && u == t - 2) ? wPre2 : 0;
    HOP_ONLY(hopWords++;)
    while (tz_status(int(w)) == kTzNone) {
      w = ld_state(&state[u + 1]);
      HOP_ONLY(hopLoads++;)
      if (tz_status(int(w)) != kTzNone)
        break;
      HOP_ONLY(hopSleeps++;)
      __nanosleep(pollNs);
    }
    const int st_ = tz_status(int(w)), v = (int(w) >> 2) & 15;
    if (st_ == kTzExit) {
      HOP_ONLY(hop_done();)
      return v + acc >= req;
    }
    if (st_ == kTzClassified) {
      const unsigned long long L = w >> 6;
      for (int i = v - 1; i >= 0; i--) {
        const int pos = acc + (v - i);
        if (pos > req) {
          HOP_ONLY(hop_done();)
          return true;
        }
        const int code = int((L >> (6 * i)) & 63);
        if (code >= 3) {
          const int li = thr_decode(code);
          if (pos + li > req)
            req = pos + li;
        }
      }
    }
    acc += v;
    if (acc >= req) {
      HOP_ONLY(hop_done();)
      return true;
    }
    u--;
  }
}

// The block kernel is compiled three times.  What a block decides per
// configuration -- encoder or decoder, integer Haar, the number of attributes
// and their rows, region qps, the root block, prediction -- is fixed for a
// launch, and the kernel is long enough for instruction fetch to matter: the
// two variants the RDOQ encoder spends its time in carry none of the arms
// they never take.
//   kBlockRdoq2    RDOQ encoder, prediction on, no region qps, below the root,
//                  colour (rows 0-2) + a one-component attribute (row 3)
//   kBlockRdoq1    the same with one attribute of 1..3 components
//   kBlockGeneric  everything else (decoder, Haar, region qps, the root step)
enum BlockVariant { kBlockGeneric = 0, kBlockRdoq1 = 1, kBlockRdoq2 = 2 };

PCC_HD BlockVariant
block_variant(const WarpBlockArgs& a)
{
  const RahtConfig& c = a.cfg;
  if (!c.isEncoder || c.haar || c.hasQp || a.P.n == 0 || !a.predInLvl)
    return kBlockGeneric;
  if (a.numSets == 1)
    return kBlockRdoq1;
  return a.set[0].A == 3 && a.set[1].A == 1 ? kBlockRdoq2 : kBlockGeneric;
}

// processes block p (worklist rank t); called by all 32 lanes.
//
// A block's latency is what bounds a stage (blocks wait for the
// reconstruction of earlier neighbours), so the order of work is: first issue
// every load that does not depend on blocks in flight (the block's own nodes,
// the parent-stage values of all 19 neighbours fetched by 19 lanes at once,
// quantisers, the inherited DC), do all the arithmetic that needs only those,
// and only then look at the values still being produced.
template<BlockVariant V>
__device__ __forceinline__ void
warp_block(const WarpBlockArgs& a, const int p, const int t, const int lane)
{
  constexpr bool fixed = V != kBlockGeneric;
  const RahtConfig& cfg = a.cfg;
  const Stage& S = a.S;
  const Stage& P = a.P;
  const int numSets = V == kBlockRdoq2 ? 2 : V == kBlockRdoq1 ? 1 : a.numSets;
  const int A = V == kBlockRdoq2 ? 4 : cfg.A;  // component rows in use (all sets)
  const int j = lane & 7;
  const int k = lane >> 3;
  const bool act = k < A;
  // the attribute this lane's component belongs to
  const int base1 = V == kBlockRdoq2 ? 3 : a.set[0].A;  // first row of the second set
  const int si = (numSets > 1 && k >= base1) ? 1 : 0;
  const AttrSet& my = a.set[si];
  const int myA = V == kBlockRdoq2 ? (si ? 1 : 3) : my.A;
  const int myBase = V == kBlockRdoq2 ? (si ? 3 : 0) : my.base;
  const int kk = k - myBase;                                     // component within its set
  const uint32_t members = ((1u << (8 * myA)) - 1) << (8 * myBase);  // lanes of the set
  // lanes of unused rows form a group of their own in the per-set reductions
  const uint32_t group = V == kBlockRdoq2 ? members : act ? members : ~((1u << (8 * A)) - 1);
  const bool speaker = lane == 8 * myBase;  // publishes the set's zero-run words
  const bool root = !fixed && P.n == 0;
  const bool haar = !fixed && cfg.haar != 0;
  const bool ext = cfg.ext != 0;
  const bool enc = fixed || cfg.isEncoder != 0;
  const bool rdoq = enc && !haar;
  const bool hasQp = !fixed && cfg.hasQp;
  const bool predInLvl = fixed || a.predInLvl;
  HOP_ONLY(long long hopT0 = clock64(), hopT1 = hopT0, hopT2 = hopT0; int hopPolls = 0;)
  HOP_STAT(kHopBlocks, 1);

  const int c0 = root ? 0 : P.first[p];
  uint32_t occ;
  if (root) {
    uint32_t bit = lane < S.n ? 1u << int((S.key[lane] >> S.level) & 7) : 0u;
    occ = __reduce_or_sync(0xffffffffu, bit);
  } else {
    occ = P.occ[p];
  }
  const bool present = (occ >> j) & 1;
  const int cidx = c0 + __popc(occ & ((1u << j) - 1));

  //-- prediction gating: neighbour indices and count come from k_block_geom;
  //   lane i < 19 fetches what the prediction needs of neighbour i
  bool enablePred = false;
  // reconstruction of the neighbours at the parent stage: lane (k, m) holds
  // component k of neighbours m, m + 8 and m + 16, so that a lane gets the
  // component it needs of neighbour i with one exchange (from lane (k, i & 7))
  int64_t nvr0 = 0, nvr1 = 0, nvr2 = 0;
  uint32_t nocc = 0;                  // its occupancy, if its children may be used
  int nfirst = 0;                     // and its first child
  uint32_t validMask = 0;             // neighbours that contribute (to this lane's attribute)
  uint32_t validAny = 0;              // ... to any attribute
  int nq = -1;                        // its index in the parent stage
  if (predInLvl) {
    const int g = lane < kGeomStride ? a.geom[size_t(t) * kGeomStride + lane] : -1;
    const int count = __shfl_sync(0xffffffffu, g, 19) & 0xff;
    nq = lane < 19 ? g : -1;
    enablePred = count >= cfg.thr1 && __shfl_sync(0xffffffffu, g, 0) >= 0;
    if (enablePred) {
      const int parentOnly = cfg.subnode ? 7 : 19;
      const int q0 = __shfl_sync(0xffffffffu, nq, j);
      const int q1 = __shfl_sync(0xffffffffu, nq, j + 8);
      const int q2 = __shfl_sync(0xffffffffu, nq, j + 16);  // (lanes 19..23 hold -1)
      if (act) {
        if (q0 >= 0)
          nvr0 = P.rec[size_t(q0) * A + k];
        if (q1 >= 0)
          nvr1 = P.rec[size_t(q1) * A + k];
        if (q2 >= 0)
          nvr2 = P.rec[size_t(q2) * A + k];
      }
      if (lane >= parentOnly && nq >= 0 && nq < p) {
        nocc = P.occ[nq];
        nfirst = P.first[nq];
      }
      // neighbours whose first component is out of range of the block's own
      // parent are ignored (RAHT.cpp:392-404): one test per attribute, on the
      // row of its first component
      const int64_t self = shfl_i64(nvr0, lane & 24);
      const int64_t limLow = 2 * self, limHigh = 25 * self;
      const bool ok0 = q0 >= 0 && (j == 0 || (10 * nvr0 > limLow && 10 * nvr0 < limHigh));
      const bool ok1 = q1 >= 0 && 10 * nvr1 > limLow && 10 * nvr1 < limHigh;
      const bool ok2 = q2 >= 0 && 10 * nvr2 > limLow && 10 * nvr2 < limHigh;
      const uint32_t b0 = __ballot_sync(0xffffffffu, ok0);
      const uint32_t b1 = __ballot_sync(0xffffffffu, ok1);
      const uint32_t b2 = __ballot_sync(0xffffffffu, ok2);
      auto row_mask = [&](int row) {
        const int sh = 8 * row;
        return ((b0 >> sh) & 0xffu) | ((b1 >> sh) & 0xffu) << 8 | ((b2 >> sh) & 0x7u) << 16;
      };
      validMask = row_mask(0);
      validAny = validMask;
      if (numSets > 1) {
        const uint32_t valid1 = row_mask(base1);
        validAny |= valid1;
        if (si)
          validMask = valid1;
      }
    }
  }

  //-- the block's own nodes
  const int w0 = present ? S.weight[cidx] : 0;
  int nodeQp0 = 0, nodeQp1 = 0;
  if (hasQp) {
    if (root) {
      if (lane == 0)
        descend_qps(S, 0, S.n, nullptr);
      __syncwarp();
    }
    if (present) {
      nodeQp0 = S.qpDown[2 * cidx] >> 4;
      nodeQp1 = S.qpDown[2 * cidx + 1] >> 4;
    }
  }
  int64_t buf = 0;
  if (enc && act && present)
    buf = fx_from_int(S.attr[size_t(cidx) * A + k]);
  int64_t dc = 0;  // inherited from the parent (RAHT.cpp:1726-1733)
  if (!root && j == 0 && act)
    dc = P.recUs[size_t(p) * A + k];
  if (!predInLvl && root && present && k == 0)
    S.nn[cidx] = 19;

  //-- quantisers of coefficient j (the encoder never reaches this kernel with
  //   AC qp offsets, so the RDOQ test and the quantisation share them)
  Quantizer qz[2];
  {
    LayerQp lq;
    lq.luma = my.qt->layers[my.qpLayer][0];
    lq.chromaOffset = my.qt->layers[my.qpLayer][1];
    lq.maxQp = my.maxQp;
    lq.fixedPointQpOffset = my.fixedPointQpOffset;
    int off0 = nodeQp0, off1 = nodeQp1;
    if (j && my.acLayer < my.numAcLayers) {
      off0 += my.qt->acQps[my.acLayer][j - 1][0];
      off1 += my.qt->acQps[my.acLayer][j - 1][1];
    }
    make_quantizers(lq, off0, off1, qz);
  }
  // RDOQ: the reciprocal of the lane's lambda (RAHT.cpp:1601-1606) for
  // rdoq_code, ready before the values the block waits for
  auto rdoq_lambda = [&]() {
    const int64_t l0 = qz[0].scale(1);
    return l0 * l0 * (myA == 1 ? 25 : 35);
  };
  const float invLambda = rdoq ? 1.0f / float(rdoq_lambda()) : 0.f;

  //-- weight tree and butterfly constants (mkWeightTree + RahtKernel)
  Bfly bf[3];
  int wcur = w0;
#pragma unroll
  for (int s = 0; s < 3; s++) {
    const int d = 1 << s;
    const int wp = __shfl_xor_sync(0xffffffffu, wcur, d);
    const bool lo = !(j & d);
    const int wl = lo ? wcur : wp;
    const int wr = lo ? wp : wcur;
    bf[s].lo = lo;
    bf[s].both = wl && wr;
    bf[s].swap = !wl && wr;
    bf[s].a = bf[s].b = 0;
    if (bf[s].both && !haar) {
      if (wl == 1 && wr == 1) {
        bf[s].a = a.ab11a;
        bf[s].b = a.ab11b;
      } else {
        const RahtAB ab = raht_ab_shared(wl, wr);
        bf[s].a = ab.a;
        bf[s].b = ab.b;
      }
    }
    wcur = (lo || bf[s].both) ? wl + wr : 0;
  }
  const int wfin = wcur;  // weights[24 + j]

  // 1/sqrt(w) scaling of this lane's child (used for the sums and the store)
  int rsShift = 0;
  int64_t rsMul = 0;
  if (!haar && w0 > 1) {
    rsShift = w0 > 1024 ? ilog2_u64(uint64_t(w0 - 1)) >> 1 : 0;
    rsMul = int64_t(irsqrt64(uint64_t(w0)) >> (40 - rsShift - kFracBits));
  }

  //-- encoder: normalise and transform the sums
  if (enc) {
    if (rsMul)
      buf = fx_mul(buf >> rsShift, rsMul);
#pragma unroll
    for (int s = 0; s < 3; s++)
      buf = bfly_fwd(buf, bf[s], 1 << s, haar);
  }

  //-- coefficients: lane (j, k) owns coefficient j of component k
  const bool exists = j == 0 ? root : wfin != 0;
  const uint32_t existsMask = __ballot_sync(0xffffffffu, exists) & 0xffu;
  // bit i' set in before(j): coefficient i' precedes j in scan order 0,4,2,1,6,5,3,7
  const uint32_t before =
    j == 0 ? 0x00u : j == 4 ? 0x01u : j == 2 ? 0x11u : j == 1 ? 0x15u
    : j == 6 ? 0x17u : j == 5 ? 0x57u : j == 3 ? 0x77u : 0x7fu;
  const int ncoef = __popc(existsMask);
  const int myPos = __popc(existsMask & before);
  const int64_t coefPos = a.coefBase + c0 - (root ? 0 : p) + myPos;
  // decoder: the coefficient comes from HBM and depends on nothing but the
  // block's position: fetched now, not after the wait for the neighbours
  int32_t qcIn = 0;
  if (!enc && exists && act)
    qcIn = my.coef[kk * my.coefStride + coefPos];

  //-- prediction (intraDcPred)
  int64_t pred = 0;
  if (enablePred) {
    int wsum = -1;
    const int64_t fracMul = ext ? 1 : (int64_t(1) << kFracBits);
    // parent-stage contributions; note which neighbours feed child values
    uint32_t childNb = 0;
    uint32_t vm = validAny;
    while (vm) {
      const int i = __ffs(vm) - 1;
      vm &= vm - 1;
      const bool counts = (validMask >> i) & 1;  // for this lane's attribute
      const uint32_t no = __shfl_sync(0xffffffffu, nocc, i);
      const int64_t src = i < 8 ? nvr0 : i < 16 ? nvr1 : nvr2;
      const int64_t mine = shfl_i64(src, (lane & 24) | (i & 7));
      const uint32_t mask = uint32_t(neigh_mask(i)) & occ;
      uint32_t cmask = 0;
      if (no) {  // only fetched for i >= parentOnly && q < p
        const int ii = i - 7;
        const int sh = occu_shift(ii);
        cmask = (ii < 9 ? (no >> sh) : (no << sh)) & mask & 0xffu;
      }
      if (cmask)
        childNb |= 1u << i;
      if (counts && ((mask >> j) & 1)) {
        if ((cmask >> j) & 1) {
          wsum += cfg.predWeightChild[i - 7];
        } else {
          const int wp = cfg.predWeightParent[i];
          wsum += wp;
          pred += mine * (wp * fracMul);
        }
      }
    }
    int64_t div = 0, sq = 0;
    if (present && act) {
      const int d = wsum + 1;
      div = (32768 + d / 2) / d;
      if (!haar && w0 > 1)
        sq = int64_t(isqrt64(uint64_t(w0) << (2 * kFracBits)));
    }
    // child-stage contributions, produced by earlier blocks of this stage: the
    // loads of up to four neighbours go out together, then whatever has not
    // been produced yet is polled
    HOP_CLOCK(hopT0);
    uint32_t cm = childNb;
    while (cm) {
      int64_t v[4];
      const int64_t* ad[4];
      int wc[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        ad[u] = nullptr;
        v[u] = 0;
        wc[u] = 0;
        if (cm) {
          const int i = __ffs(cm) - 1;
          cm &= cm - 1;
          const uint32_t no = __shfl_sync(0xffffffffu, nocc, i);
          const int cfirst = __shfl_sync(0xffffffffu, nfirst, i);
          const int ii = i - 7;
          const int sh = occu_shift(ii);
          const int shift = ii < 9 ? sh : -sh;
          const uint32_t cmask =
            (ii < 9 ? (no >> sh) : (no << sh)) & uint32_t(neigh_mask(i)) & occ & 0xffu;
          if (act && ((cmask >> j) & 1) && ((validMask >> i) & 1)) {
            const int c = cfirst + __popc(no & ((1u << (j + shift)) - 1));
            ad[u] = &S.rec[size_t(c) * A + k];
            v[u] = ld_rec(ad[u]);
            wc[u] = cfg.predWeightChild[ii];
          }
        }
      }
      // wait for all of them at once (the loop is uniform over the warp)
      for (;;) {
        bool pending = false;
#pragma unroll
        for (int u = 0; u < 4; u++)
          pending |= ad[u] && v[u] == kRecNotReady;
        if (!__any_sync(0xffffffffu, pending))
          break;
        HOP_ONLY(hopPolls++;)
        __nanosleep(a.pollNs);
#pragma unroll
        for (int u = 0; u < 4; u++)
          if (ad[u] && v[u] == kRecNotReady)
            v[u] = ld_rec(ad[u]);
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        pred += v[u] * (wc[u] * fracMul);
    }
    HOP_CLOCK(hopT1);
    HOP_STAT(kHopChildCycles, hopT1 - hopT0);
    HOP_STAT(kHopChildPolls, hopPolls);
    if (present && act) {
      int64_t v = fx_mul(pred, div);
      if (haar)
        v = (v >> kFracBits) << kFracBits;
      else if (w0 > 1)
        v = fx_mul(v, sq);
      pred = v;
    } else {
      pred = 0;
    }
#pragma unroll
    for (int s = 0; s < 3; s++)
      pred = bfly_fwd(pred, bf[s], 1 << s, haar);
  }

  // The zero-run words of the two blocks before this one, asked for as soon
  // as the neighbours' values have arrived: on a chain of adjacent blocks the
  // predecessor has just published its final word, and the round trip to L2
  // overlaps the arithmetic up to the block's own classification instead of
  // following it.
  HOP_ONLY(if (!enablePred) hopT1 = clock64();)
  unsigned long long wPre1 = 0, wPre2 = 0;
  if (rdoq && act) {
    if (t >= 1)
      wPre1 = ld_state(&my.state[t]);
    if (t >= 2)
      wPre2 = ld_state(&my.state[t - 1]);
  }

  if (enc && enablePred && exists)
    buf -= pred;

  // the coefficient of this lane before RDOQ (encoder)
  int64_t qcMine = 0;
  if (enc && exists && act)
    qcMine = qz[kk < 1 ? kk : 1].quantize(fx_round(buf) << kAttrShift);

  bool flagMine = false;
  if (rdoq) {
    int64_t d2 = 0;
    int stat = 0;  // sum |q| (clamped to 3 per component) << 16 | sum of lut_log
    if (exists && act) {
      const int64_t c = fx_round(buf);
      d2 = c * c;
      const int64_t mag = qcMine < 0 ? -qcMine : qcMine;
      stat = (mag > 3 ? 3 : int(mag)) << 16 | lut_log(mag);
    }
    // sums over the components of the lane's attribute: every row ends up with them
    if (numSets == 1) {
      d2 += shfl_xor_i64(d2, 8);
      d2 += shfl_xor_i64(d2, 16);
      stat += __shfl_xor_sync(0xffffffffu, stat, 8);
      stat += __shfl_xor_sync(0xffffffffu, stat, 16);
    } else if (V == kBlockRdoq2) {
      // rows 0-2 (colour) take the other two colour rows, row 3 keeps its own
      const int r1 = k < 3 ? (k + 1) % 3 : 3, r2 = k < 3 ? (k + 2) % 3 : 3;
      const int64_t dv1 = shfl_i64(d2, j + 8 * r1), dv2 = shfl_i64(d2, j + 8 * r2);
      const int sv1 = __shfl_sync(0xffffffffu, stat, j + 8 * r1);
      const int sv2 = __shfl_sync(0xffffffffu, stat, j + 8 * r2);
      if (k < 3) {
        d2 += dv1 + dv2;
        stat += sv1 + sv2;
      }
    } else {
      int64_t d2s = 0;
      int sts = 0;
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int64_t dv = shfl_i64(d2, j + 8 * r);
        const int sv = __shfl_sync(0xffffffffu, stat, j + 8 * r);
        if (r >= myBase && r < myBase + myA) {
          d2s += dv;
          sts += sv;
        }
      }
      d2 = d2s;
      stat = sts;
    }
    const int aq = stat >> 16, rc = stat & 0xffff;
    int code = kCodeZero;
    if (exists) {
      if (aq >= 3) {
        code = kCodeHard;
      } else if (aq > 0) {
        code = rdoq_code(d2, rdoq_lambda(), invLambda, rc);
      }
    }
    flagMine = code == kCodeRemoved;
    // the block's coefficients by scan position (the rows hold the same values)
    const uint32_t softM = __reduce_or_sync(group, exists && code >= 3 ? 1u << myPos : 0u);
    const uint32_t hardM =
      __reduce_or_sync(group, exists && code == kCodeHard ? 1u << myPos : 0u);
    const bool hasS = softM != 0, hasH = hardM != 0;
    unsigned long long codes = 0;
    if (hasS) {
      const uint32_t lo =
        __reduce_or_sync(group, exists && myPos < 5 ? uint32_t(code) << (6 * myPos) : 0u);
      const uint32_t hi =
        __reduce_or_sync(group, exists && myPos >= 5 ? uint32_t(code) << (6 * (myPos - 5)) : 0u);
      codes = lo | (unsigned long long)hi << 30;
    }

    // publish what is known without looking at any other block
    if (hasH) {
      // the run after the last coefficient that always resets it
      const int lastH = 31 - __clz(hardM);
      int e = 0, prev = lastH + 1;
      uint32_t sm = softM & ~((2u << lastH) - 1);
      while (sm) {
        const int m = __ffs(sm) - 1;
        sm &= sm - 1;
        e += m - prev;
        e = e >= thr_decode(int((codes >> (6 * m)) & 63)) ? e + 1 : 0;
        prev = m + 1;
      }
      e += ncoef - prev;
      if (speaker)
        st_state(&my.state[t + 1], state_pack(kTzExit, e, 0));
    } else if (!hasS) {
      if (speaker)
        st_state(&my.state[t + 1], state_pack(kTzTransparent, ncoef, 0));
    } else if (speaker) {
      st_state(&my.state[t + 1], state_pack(kTzClassified, ncoef, codes));
    }

    HOP_CLOCK(hopT2);
    HOP_STAT(kHopClassifyCycles, hopT2 - hopT1);

    // resolve this block's own decisions (each lane for its attribute): only
    // coefficients with a finite threshold need the run length, everything
    // between them extends it
    if (hasS) {
      bool linked = true;  // the run still reaches back beyond the block
      int z = 0;           // its length inside the block while linked
      int tl = 0;          // run length since the last reset inside the block
      int prev = 0;
      uint32_t ev = softM | hardM;
      while (ev) {
        const int m = __ffs(ev) - 1;
        ev &= ev - 1;
        if (linked)
          z += m - prev;
        else
          tl += m - prev;
        prev = m + 1;
        bool f = false;
        if ((softM >> m) & 1) {
          const int th = thr_decode(int((codes >> (6 * m)) & 63));
          if (linked) {
            HOP_ONLY(const long long hopTz = clock64();)
            f = tz_run_at_least(my, a.stageIdx, a.pollNs, t, th - z, wPre1, wPre2);
            HOP_CLOCK(hopT2);
            HOP_STAT(kHopTzCalls, 1);
            HOP_STAT(kHopTzCycles, hopT2 - hopTz);
          } else
            f = tl >= th;
        }
        if (linked) {
          if (f)
            z++;
          else {
            linked = false;
            tl = 0;
          }
        } else {
          tl = f ? tl + 1 : 0;
        }
        if (m == myPos)
          flagMine = f;
      }
      tl += ncoef - prev;
      if (!hasH && speaker)
        st_state(&my.state[t + 1], linked ? state_pack(kTzTransparent, ncoef, 0)
                                          : state_pack(kTzExit, tl, 0));
    }
  }

  HOP_ONLY(if (!rdoq) hopT2 = hopT1;)

  //-- quantise / dequantise (RAHT.cpp:1672-1723)
  int64_t qc = 0;
  if (exists && act) {
    const Quantizer& qk = qz[kk < 1 ? kk : 1];
    qc = enc ? (flagMine ? 0 : qcMine) : qcIn;
    pred += fx_from_int(div_exp2_round_half_up(qk.scale(qc), kAttrShift));
  }

  //-- DC from the parent, inverse transform, store (RAHT.cpp:1726-1806)
  if (!root && j == 0 && act)
    pred = ext ? dc : dc * (int64_t(1) << (kFracBits - 2));
#pragma unroll
  for (int s = 2; s >= 0; s--)
    pred = bfly_inv(pred, bf[s], 1 << s, haar);
  // what later blocks of this stage wait for goes out first; the values only
  // the next stage and the caller read follow
  if (present && act) {
    int64_t v = pred;
    if (rsMul)
      v = fx_mul(v >> rsShift, rsMul);
    st_rec(&S.rec[size_t(cidx) * A + k], ext ? v : fx_round(v));
  }
  HOP_STAT(kHopTailCycles, clock64() - hopT2);
  if (present && act)
    S.recUs[size_t(cidx) * A + k] = ext ? pred : fx_round(pred * 4);
  if (enc && exists && act)
    my.coef[kk * my.coefStride + coefPos] = int32_t(qc);
}

// Geometry-only part of a stage, one warp per transforming block, fully
// parallel: prediction gating (RAHT.cpp:1391-1432) and the 18 bounded
// neighbour searches of findNeighbours (RAHT.cpp:299-368), one per lane.
// Output per worklist entry t: geom[t*20 + i] = parent-stage index of
// neighbour i (i = 0 is the block's own parent) or -1; geom[t*20 + 19] = the
// neighbour count handed to the children (numParentNeigh).  A block whose
// grandparent count fails threshold0 gets index -1 in slot 0 (no search).
__global__ void __launch_bounds__(256)
k_block_geom(const WarpBlockArgs a)
{
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (t >= *a.count)
    return;
  const RahtConfig& cfg = a.cfg;
  const Stage& S = a.S;
  const Stage& P = a.P;
  const int p = a.worklist[t];
  const uint32_t occ = P.occ[p];
  int pidx = -1;
  int count = 0;
  if (P.nn[p] >= cfg.thr0) {
    const int plevel = S.level + 3;
    const int64_t cur = P.key[p] >> plevel;
    const int64_t base = int64_t(morton3d_add(uint64_t(cur), ~uint64_t(0)));
    if (lane == 0)
      pidx = p;
    else if (lane < 19 && (occ & neigh_mask(lane)))
      pidx = find_parent_neighbour(P, p, plevel, cur, base, lane, cfg.searchRange);
    count = __popc(__ballot_sync(0xffffffffu, pidx >= 0));
  }
  // same-stage dependencies: neighbour i >= 7 precedes the block, transforms
  // (a single-child block is passed through before the stage starts) and one
  // of its children is read by the sub-node prediction (RAHT.cpp:370-415)
  bool dep = false;
  if (cfg.subnode && count >= cfg.thr1 && lane >= 7 && lane < 19 && pidx >= 0 && pidx < p) {
    const int ii = lane - 7;
    const int sh = occu_shift(ii);
    const uint32_t nocc = P.occ[pidx];
    const uint32_t cmask = (ii < 9 ? (nocc >> sh) : (nocc << sh)) & uint32_t(neigh_mask(lane)) & occ & 0xffu;
    dep = cmask != 0 && P.first[pidx + 1] - P.first[pidx] >= 2;
  }
  const uint32_t depMask = (__ballot_sync(0xffffffffu, dep) >> 7) & 0xfffu;
  if (lane < 19)
    a.geom[size_t(t) * kGeomStride + lane] = pidx;
  else if (lane == 19)
    a.geom[size_t(t) * kGeomStride + 19] = count | int(depMask << 8);
  // the count is inherited by the children's blocks at the next stage
  if (lane < 8 && ((occ >> lane) & 1))
    S.nn[P.first[p] + __popc(occ & ((1u << lane) - 1))] = count;
}

// Tickets are claimed in ascending order; ticket i runs worklist entry i
// (Morton = coding order) or, with a wavefront schedule, entry order[i].  Either
// way everything a block may wait for has a lower ticket, i.e. is owned by a
// running warp.
template<BlockVariant V>
__global__ void __launch_bounds__(kWarpBlockThreads, PCCB200_BLOCK_MIN_CTAS)
k_block_warp(const WarpBlockArgs a, unsigned long long* ticket)
{
  const int lane = threadIdx.x & 31;
  const int n = *a.count;
  for (;;) {
    unsigned long long base = 0;
    if (lane == 0)
      base = atomicAdd(ticket, 1ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base >= (unsigned long long)n)
      return;
    const int t = a.order ? a.order[base] - a.orderBase : int(base);
    const int p = a.worklist ? a.worklist[t] : 0;
    warp_block<V>(a, p, t, lane);
  }
}

// A gang: several coding units (slices or frames -- independent chains with
// their own trees, tickets and zero-run streams) in ONE launch.  A textured
// unit is bound by the latency of its own chain and keeps only a handful of
// warps busy, so throughput comes from the number of chains in flight; a
// stream carries one chain, a gang launch carries as many as it has entries.
// CTA c serves entry c % numUnits (its arguments are copied to shared memory
// once); within a unit everything is as in k_block_warp.
struct GangEntry {
  WarpBlockArgs a;
  unsigned long long* ticket;
};

template<BlockVariant V>
__global__ void __launch_bounds__(kWarpBlockThreads, PCCB200_BLOCK_MIN_CTAS)
k_block_warp_gang(const GangEntry* __restrict__ tab, const int numUnits)
{
  __shared__ GangEntry se;
  {
    static_assert(sizeof(GangEntry) % sizeof(uint32_t) == 0, "copied by words");
    const uint32_t* src = reinterpret_cast<const uint32_t*>(tab + blockIdx.x % numUnits);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&se);
    for (int i = threadIdx.x; i < int(sizeof(GangEntry) / sizeof(uint32_t)); i += blockDim.x)
      dst[i] = src[i];
  }
  __syncthreads();
  const WarpBlockArgs& a = se.a;
  unsigned long long* const ticket = se.ticket;
  const int lane = threadIdx.x & 31;
  const int n = *a.count;
  for (;;) {
    unsigned long long base = 0;
    if (lane == 0)
      base = atomicAdd(ticket, 1ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base >= (unsigned long long)n)
      return;
    const int t = a.order ? a.order[base] - a.orderBase : int(base);
    const int p = a.worklist ? a.worklist[t] : 0;
    warp_block<V>(a, p, t, lane);
  }
}

__device__ __forceinline__ int
ld_relaxed_i32(const int* p)
{
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void
st_relaxed_i32(int* p, int v)
{
  asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace pccb200
