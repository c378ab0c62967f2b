// lod_core.cuh — per-item bodies of the level-of-detail build of the
// predicting / lifting transforms (intra; scalable lifting included).
//
// Replaces (paths relative to the TMC13 tree):
//   buildPredictorsFast            tmc3/PCCTMC3Common.h:2300-2469
//   subsampleByDistance/ByDecimation/ByOctree   tmc3/PCCTMC3Common.h:1984-2250
//   computeNearestNeighbors        tmc3/PCCTMC3Common.h:1147-1953
//   updateNearestNeigh*            tmc3/PCCTMC3Common.h:944-1143
//   updatePredictors               tmc3/PCCTMC3Common.h:2273-2296
//   PCCPredictor::computeWeights / blendWeights  tmc3/PCCTMC3Common.h:589-693
//   AttributeLods::generate        tmc3/AttributeCommon.cpp:45-72
//
// The reference walks the refined points of a LoD in Morton order carrying
// cursors and a hash atlas (it is NOT nanoflann: an L1-metric search over 27
// atlas cells, then a bounded window with bounding-box pruning, with
// visit-order-dependent tie breaking).  Here every query is one thread and a
// pure function of (query, Morton-sorted retained list): cell ranges are
// binary searches, the window walk uses a 3-level bounding-box hierarchy in
// HBM, the candidate visit order of the reference is replayed exactly, and
// the reference's one stateful quirk (the atlas fill cursor stalls for good
// once an atlas holding retained points holds no query) is reproduced from a
// per-LoD reduction (`StuckAtlasFn`).  Distance subsampling — a greedy,
// order-dependent selection — runs as a dataflow over cells in Morton order
// (`SubsampleDistanceFn`, ordered executor launch).
#pragma once

#include "pcc_arith.cuh"
#include "raht_core.cuh"

namespace pccb200 {

struct LodConfig {
  int numDetailLevels;
  int decimation;  // 0 distance, 1 periodic, 2 centroid
  int samplingPeriod[PCCB200_MAX_LODS];
  int dist2;
  int numNeighbours;
  int interRange;
  int intraRange;
  int intraSkipLayers;
  int distribution;
  int bias[3];
  int blending;
  int maxNeighRange;  // scalable lifting: neighbour pruning range, else 0 (no pruning)
};

// sorted voxels (Morton order, ties by point index)
struct Voxels {
  int n;
  const int64_t* code;
  const int32_t* pos;   // n*3, original positions
  const int32_t* bpos;  // n*3, positions * lodNeighBias
  const int32_t* pidx;  // original point index
};

struct Box {
  int32_t mn[3], mx[3];
};

PCC_HD int32_t
box_dist1(const Box& b, const int32_t* p)
{
  int32_t s = 0;
  for (int k = 0; k < 3; k++) {
    int32_t a = b.mn[k] - p[k], c = p[k] - b.mx[k];
    int32_t d = a > 0 ? a : 0;
    s += c > d ? c : d;
  }
  return s;
}

// level l box i covers entries [i << 5(l+1), ...) of `list`
struct BoxLevelFn {
  const int32_t* bpos;
  const uint32_t* list;  // level 0: entry list; else null
  const Box* lower;      // level > 0: boxes of the level below
  int count;             // entries (level 0) or lower boxes
  Box* out;
  PCC_HD void operator()(int64_t b) const
  {
    Box r;
    for (int k = 0; k < 3; k++) {
      r.mn[k] = INT32_MAX;
      r.mx[k] = INT32_MIN;
    }
    int lo = int(b) << 5, hi = lo + 32 < count ? lo + 32 : count;
    for (int i = lo; i < hi; i++) {
      if (list) {
        const int32_t* p = &bpos[size_t(list[i]) * 3];
        for (int k = 0; k < 3; k++) {
          r.mn[k] = p[k] < r.mn[k] ? p[k] : r.mn[k];
          r.mx[k] = p[k] > r.mx[k] ? p[k] : r.mx[k];
        }
      } else {
        for (int k = 0; k < 3; k++) {
          r.mn[k] = lower[i].mn[k] < r.mn[k] ? lower[i].mn[k] : r.mn[k];
          r.mx[k] = lower[i].mx[k] > r.mx[k] ? lower[i].mx[k] : r.mx[k];
        }
      }
    }
    out[b] = r;
  }
};

struct BoxHierarchy {
  const Box* lvl[3];
};

//============================================================================
// subsampling

// periodic: every period-th entry of `input` is retained
struct SubsamplePeriodicFn {
  const uint32_t* input;
  uint32_t* retained;
  uint32_t* indexes;  // already offset to the LoD's start
  int period;
  PCC_HD void operator()(int64_t i) const
  {
    if (period <= 0) {
      indexes[i] = input[i];
      return;
    }
    int64_t q = i / period;
    if (i - q * period == 0)
      retained[q] = input[i];
    else
      indexes[i - (q + 1)] = input[i];
  }
};

// group structure shared by the distance and centroid subsampling: cells are
// maximal runs of input entries with equal (code >> shift)
struct CellHead {
  const int64_t* code;
  const uint32_t* input;
  int shift;
  PCC_HD bool operator()(int64_t i) const
  {
    return i == 0 || (code[input[i]] >> shift) != (code[input[i - 1]] >> shift);
  }
};
struct CellEmit {
  int32_t* first;
  PCC_HD void operator()(int64_t rank, int64_t i) const { first[rank] = int32_t(i); }
};

PCC_HD int64_t
norm2_3(const int32_t* a, const int32_t* b)
{
  int64_t s = 0;
  for (int k = 0; k < 3; k++) {
    int64_t d = int64_t(a[k]) - b[k];
    s += d * d;
  }
  return s;
}

PCC_HD int64_t
norm1_3(const int32_t* a, const int32_t* b)
{
  int32_t s = 0;  // int32 arithmetic like Vec3<int32_t>::getNorm1
  for (int k = 0; k < 3; k++) {
    int32_t d = a[k] - b[k];
    s += d < 0 ? -d : d;
  }
  return s;
}

// index of the cell with code `cell` in the sorted cell list, or -1
PCC_HD int
find_cell(const int64_t* code, const uint32_t* input, const int32_t* cellFirst, int nCells,
          int shift, int64_t cell)
{
  int lo = 0, hi = nCells;
  while (lo < hi) {
    int m = (lo + hi) >> 1;
    if ((code[input[cellFirst[m]]] >> shift) < cell)
      lo = m + 1;
    else
      hi = m;
  }
  return (lo < nCells && (code[input[cellFirst[lo]]] >> shift) == cell) ? lo : -1;
}

// Distance subsampling (subsampleByDistance, PCCTMC3Common.h:1984-2085): in
// Morton order a point is dropped if its cell already holds the most recently
// retained point, or if a retained point of one of 20 listed neighbour cells
// (same atlas) lies within the radius; otherwise it is retained.  Each cell
// ends up with at most one retained point, decided by the cell's own points in
// order and by the decisions of Morton-EARLIER neighbour cells only: one work
// item per cell, claimed in Morton order, spinning on the decision words of
// earlier cells.
constexpr int kCellUndecided = -2;
constexpr int kCellNone = -1;

struct SubsampleDistanceFn {
  Voxels v;
  const uint32_t* input;
  int nInput;
  const int32_t* cellFirst;  // nCells + 1
  int nCells;
  int shiftBits0;            // dist2 + lod
  int* decision;             // per cell: input position of its retained point
  uint8_t* keep;             // per input position: 1 = retained
  PCC_HD void operator()(int64_t cb) const
  {
    const int c = int(cb);
    const int sb3 = 3 * (shiftBits0 + 1);
    const int atlasBit = sb3 + 21 < 63 ? sb3 + 21 : 63;
    const int64_t radius2 = int64_t(3) << (shiftBits0 << 1);
    const uint8_t kOff[20] = {7,  3,  5,  6,  12, 10, 17, 20, 34, 33,
                              4,  2,  1,  24, 40, 48, 32, 16, 8,  0};
    const int i0 = cellFirst[c], i1 = cellFirst[c + 1];
    const int64_t code0 = v.code[input[i0]];
    const int64_t cell = code0 >> sb3;
    const int64_t atlasId = code0 >> atlasBit;
    const uint64_t base = morton3d_add(uint64_t(cell), ~uint64_t(0));
    // retained points of the earlier neighbour cells
    int nb[19];
    int nnb = 0;
    for (int n = 1; n < 20; n++) {
      const int64_t nc = int64_t(morton3d_add(base, kOff[n]));
      if ((nc >> 21) != atlasId)
        continue;
      int q = find_cell(v.code, input, cellFirst, nCells, sb3, nc);
      if (q < 0 || q >= c)
        continue;  // absent, or later in Morton order: nothing retained there yet
      if ((v.code[input[cellFirst[q]]] >> atlasBit) != atlasId)
        continue;
      int d;
      while ((d = ld_acquire(&decision[q])) == kCellUndecided)
        spin_pause();
      if (d >= 0)
        nb[nnb++] = int(input[d]);
    }
    int chosen = kCellNone;
    for (int i = i0; i < i1; i++) {
      const int32_t* p = &v.pos[size_t(input[i]) * 3];
      bool found = false;
      for (int h = 0; h < nnb && !found; h++)
        found = norm2_3(&v.pos[size_t(nb[h]) * 3], p) <= radius2;
      keep[i] = found ? 0 : 1;
      if (!found) {
        chosen = i;
        for (int r = i + 1; r < i1; r++)
          keep[r] = 0;
        break;
      }
    }
#if defined(__CUDA_ARCH__)
    __threadfence();
#endif
    st_release(&decision[c], chosen);
  }
};

// Centroid subsampling (subsampleByOctree + ...WithCentroid,
// PCCTMC3Common.h:2089-2194).  Groups of equal (code >> q) are merged until a
// segment holds at least `period` entries; each segment retains the entry
// nearest (L1) to the segment's centroid.  Centroid decimation scans backward
// (ties: the last minimum); scalable lifting scans in the direction
// lodIndex & 1 (PCCTMC3Common.h:2230-2235), forward keeping the first minimum.
//
// The greedy segmentation is a recurrence over group ends (the next segment
// starts where the previous one closed).  Parallel form: nxt[c] = first group
// of the segment that follows a segment starting at group c (a binary search
// per group: group sizes are prefix sums); the segment starts are the groups
// reachable from group 0 through nxt, found by pointer doubling (jump tables
// nxt^(2^i), then marking from the widest jump down).
struct CentroidNextFn {
  const int32_t* cellFirst;  // group starts, nCells + 1
  int nCells;
  int period;
  int32_t* nxt;  // out; nCells = no further segment
  PCC_HD void operator()(int64_t ci) const
  {
    const int c = int(ci);
    const int g0 = cellFirst[c];
    // the segment closes at the first group whose end makes it `period`
    // long; the last group closes whatever is open
    int lo = c, hi = nCells - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cellFirst[mid + 1] - g0 >= period)
        hi = mid;
      else
        lo = mid + 1;
    }
    nxt[c] = lo + 1;
  }
};

struct JumpSquareFn {  // dst = src o src
  const int32_t* src;
  int32_t* dst;
  int nCells;
  PCC_HD void operator()(int64_t c) const
  {
    const int j = src[c];
    dst[c] = j < nCells ? src[j] : nCells;
  }
};

// marks jump[c] for every marked c.  Threads of one pass may or may not see
// marks set in the same pass: either way only groups on the path get marked,
// and every mark of the earlier passes is seen, which is what completeness needs.
struct JumpMarkFn {
  const int32_t* jump;
  uint8_t* mark;
  int nCells;
  PCC_HD void operator()(int64_t c) const
  {
    if (mark[c]) {
      const int j = jump[c];
      if (j < nCells)
        mark[j] = 1;
    }
  }
};

struct MarkPred {
  const uint8_t* mark;
  PCC_HD bool operator()(int64_t c) const { return mark[c] != 0; }
};
struct SegmentEmit {
  const int32_t* cellFirst;
  int32_t* segFirst;
  PCC_HD void operator()(int64_t rank, int64_t c) const { segFirst[rank] = cellFirst[c]; }
};

struct CentroidPickFn {
  Voxels v;
  const uint32_t* input;
  const int32_t* segFirst;
  int nodeLog2;
  bool backward;
  uint8_t* keep;
  PCC_HD void operator()(int64_t sg) const
  {
    const int g0 = segFirst[sg], g1 = segFirst[sg + 1];
    const uint32_t mask = nodeLog2 ? ~uint32_t(0) << nodeLog2 : ~uint32_t(0);
    const int size = g1 - g0;
    int32_t cen[3] = {0, 0, 0};
    for (int t = g0; t < g1; t++)
      for (int k = 0; k < 3; k++)
        cen[k] += int32_t(uint32_t(v.pos[size_t(input[t]) * 3 + k]) & mask);
    int pick = backward ? g1 - 1 : g0;
    int64_t best = INT64_MAX;
    for (int u = 0; u < size; u++) {
      const int t = backward ? g1 - 1 - u : g0 + u;
      int32_t pp[3];
      for (int k = 0; k < 3; k++)
        pp[k] = int32_t(uint32_t(v.pos[size_t(input[t]) * 3 + k]) & mask) * size;
      int64_t m = norm1_3(pp, cen);
      if (best > m) {
        best = m;
        pick = t;
      }
    }
    for (int t = g0; t < g1; t++)
      keep[t] = t == pick;
  }
};

// split `input` by the keep flags
struct KeepPred {
  const uint8_t* keep;
  int want;
  PCC_HD bool operator()(int64_t i) const { return keep[i] == want; }
};
struct ListEmit {
  const uint32_t* input;
  uint32_t* out;
  PCC_HD void operator()(int64_t rank, int64_t i) const { out[rank] = input[i]; }
};

//============================================================================
// nearest-neighbour search

struct NNState {
  int32_t li[6];
  int64_t md[6];
  int index2;
};

// updateNearestNeigh / ...ByDistanceAndDistribution (PCCTMC3Common.h:944-1069)
PCC_HD void
nn_update(NNState& s, bool distribution, int64_t d, int32_t index)
{
  if (!distribution) {
    if (d >= s.md[2])
      return;
  } else {
    if (d > s.md[2])
      return;
    if (d == s.md[2]) {
      // exact tie with the third neighbour: kept as a spare candidate
      if (s.li[5] == -1) {
        s.li[s.index2++] = index;
        if (s.index2 == 6)
          s.index2 = 3;
      }
      return;
    }
    if (s.li[2] != -1) {
      s.li[s.index2++] = s.li[2];  // the evicted third neighbour becomes a spare
      if (s.index2 == 6)
        s.index2 = 3;
    }
  }
  if (d < s.md[0]) {
    s.md[2] = s.md[1];
    s.md[1] = s.md[0];
    s.md[0] = d;
    s.li[2] = s.li[1];
    s.li[1] = s.li[0];
    s.li[0] = index;
  } else if (d < s.md[1]) {
    s.md[2] = s.md[1];
    s.md[1] = d;
    s.li[2] = s.li[1];
    s.li[1] = index;
  } else {
    s.md[2] = d;
    s.li[2] = index;
  }
}

PCC_HD void
nn_update_check(NNState& s, bool distribution, int64_t d, int32_t index)
{
  const int lim = distribution ? 6 : 3;
  for (int h = 0; h < lim; h++)
    if (s.li[h] == index)
      return;
  nn_update(s, distribution, d, index);
}

// [lo, hi) of entries of `list` whose (code >> shift) == cell
PCC_HD void
cell_range(const int64_t* code, const uint32_t* list, int n, int shift, int64_t cell, int& lo,
           int& hi)
{
  int a = 0, b = n;
  while (a < b) {
    int m = (a + b) >> 1;
    if ((code[list[m]] >> shift) < cell)
      a = m + 1;
    else
      b = m;
  }
  lo = a;
  b = n;
  while (a < b) {
    int m = (a + b) >> 1;
    if ((code[list[m]] >> shift) <= cell)
      a = m + 1;
    else
      b = m;
  }
  hi = a;
}

// The atlas fill cursor of the reference stalls at the first atlas that holds
// retained points but no query (PCCTMC3Common.h:1337-1349); from then on the
// 27-cell stage finds nothing.  One work item per retained entry: entries that
// open an atlas look that atlas up among the queries.
struct StuckAtlasFn {
  const int64_t* code;
  const uint32_t* retained;
  const uint32_t* queries;
  int nQueries;
  int atlasBit;
  unsigned long long* stuck;  // min over atlases without query (init: max)
  PCC_HD void operator()(int64_t r) const
  {
    const int64_t a = code[retained[r]] >> atlasBit;
    if (r > 0 && (code[retained[r - 1]] >> atlasBit) == a)
      return;
    int lo = 0, hi = nQueries;
    while (lo < hi) {
      int m = (lo + hi) >> 1;
      if ((code[queries[m]] >> atlasBit) < a)
        lo = m + 1;
      else
        hi = m;
    }
    if (lo < nQueries && (code[queries[lo]] >> atlasBit) == a)
      return;
#if defined(__CUDA_ARCH__)
    atomicMin(stuck, (unsigned long long)a);
#else
    if ((unsigned long long)a < *stuck)
      *stuck = (unsigned long long)a;
#endif
  }
};

struct KnnFn {
  LodConfig cfg;
  Voxels v;
  const uint32_t* retained;
  int R;
  const uint32_t* queries;  // sorted-voxel indices of the LoD's refined points
  int nQueries;
  int lod;
  BoxHierarchy hb;          // over `retained`
  BoxHierarchy hq;          // over `queries` (intra-LoD search only)
  const unsigned long long* stuck;
  int predBase;             // predictor slot of query 0 is predBase - 1
  uint32_t* indexesOut;     // LoD region of `indexes`: point index of query i
  uint32_t* p2p;            // point index -> predictor slot
  uint32_t* predCount;
  uint32_t* predIdx;        // slot*3 + h: point index of neighbour h
  uint64_t* predW;          // slot*3 + h: squared distance

  PCC_HD void window(NNState& s, const int32_t* bp, int lo, int hi, int dir) const
  {
    if (lo > hi)
      return;
    const bool dist = cfg.distribution != 0;
    const int b2lo = lo >> 15, b2hi = hi >> 15, b1lo = lo >> 10, b1hi = hi >> 10;
    const int b0lo = lo >> 5, b0hi = hi >> 5;
    for (int t2 = 0; t2 <= b2hi - b2lo; t2++) {
      const int b2 = dir > 0 ? b2lo + t2 : b2hi - t2;
      if (s.li[2] != -1 && box_dist1(hb.lvl[2][b2], bp) >= s.md[2])
        continue;
      const int a1 = b2 << 5;
      const int s1 = b1lo > a1 ? b1lo : a1, e1 = b1hi < a1 + 31 ? b1hi : a1 + 31;
      for (int t1 = 0; t1 <= e1 - s1; t1++) {
        const int b1 = dir > 0 ? s1 + t1 : e1 - t1;
        if (s.li[2] != -1 && box_dist1(hb.lvl[1][b1], bp) >= s.md[2])
          continue;
        const int a0 = b1 << 5;
        const int s0 = b0lo > a0 ? b0lo : a0, e0 = b0hi < a0 + 31 ? b0hi : a0 + 31;
        for (int t0 = 0; t0 <= e0 - s0; t0++) {
          const int b0 = dir > 0 ? s0 + t0 : e0 - t0;
          if (s.li[2] != -1 && box_dist1(hb.lvl[0][b0], bp) >= s.md[2])
            continue;
          const int a = b0 << 5;
          const int k0 = lo > a ? lo : a, k1 = hi < a + 31 ? hi : a + 31;
          for (int t = 0; t <= k1 - k0; t++) {
            const int k = dir > 0 ? k0 + t : k1 - t;
            nn_update_check(s, dist, norm1_3(bp, &v.bpos[size_t(retained[k]) * 3]), k);
          }
        }
      }
    }
  }

  PCC_HD void operator()(int64_t qi) const
  {
    const int i = int(qi);
    const bool dist = cfg.distribution != 0;
    const uint32_t index = queries[i];
    const int64_t code = v.code[index];
    const int32_t* bp = &v.bpos[size_t(index) * 3];
    NNState s;
    for (int h = 0; h < 6; h++) {
      s.li[h] = -1;
      s.md[h] = INT64_MAX;
    }
    s.index2 = 3;
    const int slot = predBase - 1 - i;
    const int32_t pointIndex = v.pidx[index];
    indexesOut[i] = uint32_t(pointIndex);
    p2p[pointIndex] = uint32_t(slot);

    const int shiftBits = 1 + cfg.dist2 + lod;
    const int sb3 = 3 * shiftBits;
    const int atlasBit = sb3 + 21 < 63 ? sb3 + 21 : 63;
    if (R) {
      int j;
      {
        int a = 0, b = R;
        while (a < b) {
          int m = (a + b) >> 1;
          if (v.code[retained[m]] <= code)
            a = m + 1;
          else
            b = m;
        }
        j = a < R - 1 ? a : R - 1;
      }
      const int64_t atlasId = code >> atlasBit;
      if ((unsigned long long)atlasId < *stuck) {
        const uint8_t kOff[27] = {7,  3,  5,  6,  35, 21, 14, 28, 42, 49, 12, 10, 17, 20,
                                  34, 33, 4,  2,  1,  56, 24, 40, 48, 32, 16, 8,  0};
        const uint64_t base = morton3d_add(uint64_t(code >> sb3), ~uint64_t(0));
        for (int n = 0; n < 27; n++) {
          const int64_t nb = int64_t(morton3d_add(base, kOff[n]));
          if ((nb >> 21) != atlasId)
            continue;
          int lo, hi;
          cell_range(v.code, retained, R, sb3, nb, lo, hi);
          for (int k = lo; k < hi; k++)
            if ((v.code[retained[k]] >> atlasBit) == atlasId)
              nn_update(s, dist, norm1_3(bp, &v.bpos[size_t(retained[k]) * 3]), k);
        }
      }
      if (s.li[2] == -1) {
        const int center = s.li[0] == -1 ? j : s.li[0];
        const int range = cfg.interRange;
        const int k0 = center - range > 0 ? center - range : 0;
        const int k1 = int64_t(center) + range < R - 1 ? center + range : R - 1;
        nn_update_check(s, dist, norm1_3(bp, &v.bpos[size_t(retained[center]) * 3]), center);
        for (int n = 1; n <= 2; n++) {
          if (center + n <= k1)
            nn_update_check(s, dist, norm1_3(bp, &v.bpos[size_t(retained[center + n]) * 3]),
                            center + n);
          if (center - n >= k0)
            nn_update_check(s, dist, norm1_3(bp, &v.bpos[size_t(retained[center - n]) * 3]),
                            center - n);
        }
        const int p1 = center + 3 < R - 1 ? center + 3 : R - 1;
        const int p0 = center - 3 > 0 ? center - 3 : 0;
        window(s, bp, p1, k1, +1);
        window(s, bp, k0, p0, -1);
      }
      // retained-list positions -> sorted-voxel indices
      for (int h = 0; h < 6; h++)
        if (s.li[h] != -1 && (h < 3 || dist))
          s.li[h] = int32_t(retained[s.li[h]]);
    }

    if (lod >= cfg.intraSkipLayers) {
      // candidates inside the same LoD: the following entries
      const int end = nQueries;
      const int k00 = i + 1;
      const int k01 = end - 1 < k00 + 2 ? end - 1 : k00 + 2;
      for (int k = k00; k <= k01; k++)
        nn_update(s, dist, norm1_3(bp, &v.bpos[size_t(queries[k]) * 3]), int32_t(queries[k]));
      const int w0 = k01 + 1;
      const int w1 = end - 1 < k00 + cfg.intraRange ? end - 1 : k00 + cfg.intraRange;
      if (w0 <= w1) {
        const int b2lo = w0 >> 15, b2hi = w1 >> 15, b1lo = w0 >> 10, b1hi = w1 >> 10;
        const int b0lo = w0 >> 5, b0hi = w1 >> 5;
        for (int b2 = b2lo; b2 <= b2hi; b2++) {
          if (s.li[2] != -1 && box_dist1(hq.lvl[2][b2], bp) >= s.md[2])
            continue;
          const int a1 = b2 << 5;
          const int s1 = b1lo > a1 ? b1lo : a1, e1 = b1hi < a1 + 31 ? b1hi : a1 + 31;
          for (int b1 = s1; b1 <= e1; b1++) {
            if (s.li[2] != -1 && box_dist1(hq.lvl[1][b1], bp) >= s.md[2])
              continue;
            const int a0 = b1 << 5;
            const int s0 = b0lo > a0 ? b0lo : a0, e0 = b0hi < a0 + 31 ? b0hi : a0 + 31;
            for (int b0 = s0; b0 <= e0; b0++) {
              if (s.li[2] != -1 && box_dist1(hq.lvl[0][b0], bp) >= s.md[2])
                continue;
              const int a = b0 << 5;
              const int h0 = w0 > a ? w0 : a, h1 = w1 < a + 31 ? w1 : a + 31;
              for (int h = h0; h <= h1; h++)
                nn_update(s, dist, norm1_3(bp, &v.bpos[size_t(queries[h]) * 3]),
                          int32_t(queries[h]));
            }
          }
        }
      }
    }

    int nc = (s.li[0] != -1) + (s.li[1] != -1) + (s.li[2] != -1);
    if (nc > cfg.numNeighbours)
      nc = cfg.numNeighbours;
    if (dist) {
      // spare candidates: distances, ordering, and the direction test that may
      // swap the third neighbour for a better placed spare
      // (PCCTMC3Common.h:1802-1903)
      const int nc1 = 3 + (s.li[3] != -1) + (s.li[4] != -1) + (s.li[5] != -1);
      for (int m = 3; m < nc1; m++)
        if (s.md[m] == INT64_MAX)
          s.md[m] = norm1_3(bp, &v.bpos[size_t(s.li[m]) * 3]);
      for (int m = 3; m < nc1; m++)
        for (int l = m + 1; l < nc1; l++)
          if (s.md[l] < s.md[m]) {
            int32_t ti = s.li[l];
            s.li[l] = s.li[m];
            s.li[m] = ti;
            int64_t td = s.md[l];
            s.md[l] = s.md[m];
            s.md[m] = td;
          }
      if (nc >= 3) {
        const int8_t kLoose[8][3] = {{3, 5, 6}, {2, 4, 7}, {1, 4, 7}, {0, 5, 6},
                                     {1, 2, 7}, {0, 3, 6}, {0, 3, 5}, {1, 2, 4}};
        int dir[6] = {-1, -1, -1, -1, -1, -1};
        int numend = 3;
        for (; numend < nc1; numend++)
          if ((s.md[numend] << 5) >= s.md[2] * 54)
            break;
        for (int h = 0; h < numend; h++) {
          const int32_t* q = &v.bpos[size_t(s.li[h]) * 3];
          dir[h] = ((q[0] - bp[0] >= 0) << 2) + ((q[1] - bp[1] >= 0) << 1) + (q[2] - bp[2] >= 0);
        }
        bool replace = true;
        int ridx = -1;
        if (dir[1] == 7 - dir[0] || dir[2] == 7 - dir[0] || dir[2] == 7 - dir[1])
          replace = false;
        for (int h = 3; replace && h < numend; h++)
          if (dir[h] == 7 - dir[0] || dir[h] == 7 - dir[1]) {
            replace = false;
            ridx = h;
          }
        const bool e01 = dir[0] == dir[1], e02 = dir[0] == dir[2], e12 = dir[1] == dir[2];
        const int8_t* ld = kLoose[dir[0]];
        auto loose = [&](int x) { return x == ld[0] || x == ld[1] || x == ld[2]; };
        if (replace) {
          if ((e02 || e12) && e01) {
            for (int h = 3; replace && h < numend; h++)
              if (loose(dir[h])) {
                replace = false;
                ridx = h;
              }
          } else if ((e02 || e12) && !e01) {
            if (!loose(dir[1]))
              for (int h = 3; replace && h < numend; h++)
                if (dir[h] != dir[0] && dir[h] != dir[1]) {
                  replace = false;
                  ridx = h;
                }
          } else if (e01) {
            if (!loose(dir[2]))
              for (int h = 3; replace && h < numend; h++)
                if (loose(dir[h])) {
                  replace = false;
                  ridx = h;
                }
          }
        }
        if (ridx >= 0)
          s.li[2] = s.li[ridx];
      }
    }
    uint64_t w[3] = {0, 0, 0};
    uint32_t ix[3] = {0, 0, 0};
    for (int h = 0; h < nc; h++) {
      ix[h] = uint32_t(v.pidx[s.li[h]]);
      w[h] = uint64_t(norm2_3(&v.bpos[size_t(s.li[h]) * 3], bp));
    }
    if (cfg.maxNeighRange > 0) {
      // scalable lifting: drop the candidates beyond the range, and every one
      // after them in candidate order (PCCTMC3Common.h:1918-1937).  Unit bias:
      // on the weights; otherwise on the unbiased positions masked to the level.
      const int64_t maxDistance = (int64_t(3) * cfg.maxNeighRange) << (2 * lod);
      const bool unitBias = cfg.bias[0] == 1 && cfg.bias[1] == 1 && cfg.bias[2] == 1;
      const uint32_t mask = lod ? ~uint32_t(0) << lod : ~uint32_t(0);
      for (int h = 1; h < nc; h++) {
        int64_t d;
        if (unitBias) {
          d = int64_t(w[h]);
        } else {
          int32_t a[3], b[3];
          for (int k = 0; k < 3; k++) {
            a[k] = int32_t(uint32_t(v.pos[size_t(index) * 3 + k]) & mask);
            b[k] = int32_t(uint32_t(v.pos[size_t(s.li[h]) * 3 + k]) & mask);
          }
          d = norm2_3(a, b);
        }
        if (uint64_t(d) > uint64_t(maxDistance)) {
          nc = h;
          break;
        }
      }
    }
    // order by squared distance (PCCTMC3Common.h:1941-1951)
    auto swp = [&](int a, int b) {
      uint64_t tw = w[a];
      w[a] = w[b];
      w[b] = tw;
      uint32_t tx = ix[a];
      ix[a] = ix[b];
      ix[b] = tx;
    };
    if (nc > 1) {
      if (w[0] > w[1])
        swp(0, 1);
      if (nc == 3 && w[1] > w[2]) {
        swp(1, 2);
        if (w[0] > w[1])
          swp(0, 1);
      }
    }
    predCount[slot] = uint32_t(nc);
    for (int h = 0; h < 3; h++) {
      predIdx[size_t(slot) * 3 + h] = ix[h];
      predW[size_t(slot) * 3 + h] = w[h];
    }
  }
};

//============================================================================
// finalisation: updatePredictors + computeWeights (+ blendWeights), and the
// coarse-to-fine ordering of `indexes`

struct FinalizePredictorFn {
  int n;
  int blending;
  const uint32_t* predCount;
  const uint32_t* predIdx;
  const uint64_t* predW;
  const uint32_t* p2p;
  const uint32_t* indexesBuild;  // in build order (fine to coarse): reversed on the fly
  const int32_t* xyz;            // original positions (blendWeights)
  pccb200_predictor* out;
  uint32_t* indexesOut;
  PCC_HD void operator()(int64_t i) const
  {
    indexesOut[i] = indexesBuild[n - 1 - i];
    uint32_t nc = predCount[i];
    uint64_t w[3];
    uint32_t ix[3];
    for (int h = 0; h < 3; h++) {
      w[h] = predW[size_t(i) * 3 + h];
      ix[h] = predIdx[size_t(i) * 3 + h];
    }
    if (nc < 2) {
      w[0] = 1;
    } else if (w[0] == 0) {
      nc = 1;
      w[0] = 1;
    }
    for (uint32_t h = 0; h < nc; h++)
      ix[h] = p2p[ix[h]];
    // computeWeights
    const uint32_t shift = 1u << 8;
    int sh = 0;
    while ((w[0] >> sh) >= shift)
      sh++;
    if (sh > 0)
      for (uint32_t h = 0; h < nc; h++)
        w[h] = (w[h] + (uint64_t(1) << (sh - 1))) >> sh;
    while (nc > 1 && w[nc - 1] >= (w[0] << 8))
      nc--;
    if (nc <= 1) {
      w[0] = shift;
    } else if (nc == 2) {
      const uint64_t d0 = w[0], d1 = w[1];
      const uint64_t w1 = uint64_t(div_approx(int64_t(d0), d0 + d1, 8));
      w[0] = shift - w1;
      w[1] = w1;
    } else {
      const uint64_t d0 = w[0], d1 = w[1], d2 = w[2];
      const uint64_t sum = d1 * d2 + d0 * d2 + d0 * d1;
      const uint64_t w2 = uint64_t(div_approx(int64_t(d0 * d1), sum, 8));
      const uint64_t w1 = uint64_t(div_approx(int64_t(d0 * d2), sum, 8));
      w[0] = shift - (w1 + w2);
      w[1] = w1;
      w[2] = w2;
    }
    if (blending && nc == 3) {
      // neighbour positions through the final (reversed) index list
      const int32_t* n0 = &xyz[size_t(indexesBuild[n - 1 - ix[0]]) * 3];
      const int32_t* n1 = &xyz[size_t(indexesBuild[n - 1 - ix[1]]) * 3];
      const int32_t* n2 = &xyz[size_t(indexesBuild[n - 1 - ix[2]]) * 3];
      const int64_t d01 = norm2_3(n0, n1), d02 = norm2_3(n0, n2), d12 = norm2_3(n1, n2);
      const int w0 = int(uint32_t(w[0])), w1 = int(uint32_t(w[1])), w2 = int(uint32_t(w[2]));
      const int b1 = d01 <= d02 ? 1 : 5;
      const int b2 = d01 <= d12 ? 5 : 1;
      const int b3 = d02 <= d12 ? 1 : 5;
      const int r0 = (w0 * 10 + w1 * (16 - 10 - b2) + w2 * b3) >> 4;
      const int r1 = (w0 * b1 + w1 * 10 + w2 * (16 - 10 - b3)) >> 4;
      w[0] = uint64_t(r0);
      w[1] = uint64_t(r1);
      w[2] = uint64_t(256 - r0 - r1);
    }
    pccb200_predictor p;
    p.neighbor_count = nc;
    for (uint32_t h = 0; h < 3; h++) {
      p.predictor_index[h] = h < nc ? ix[h] : 0;
      p.weight[h] = h < nc ? uint32_t(w[h]) : 0;
    }
    out[i] = p;
  }
};

// scalable lifting: the biased positions of a level are the positions masked
// to its node grid, times lodNeighBias (clacIntermediatePosition,
// PCCTMC3Common.h:926-940 and :1230-1236)
struct BiasMaskFn {
  const int32_t* pos;
  int bias[3];
  int nodeLog2;
  int32_t* bpos;
  PCC_HD void operator()(int64_t i) const
  {
    const uint32_t mask = nodeLog2 ? ~uint32_t(0) << nodeLog2 : ~uint32_t(0);
    for (int k = 0; k < 3; k++)
      bpos[i * 3 + k] = int32_t(uint32_t(pos[i * 3 + k]) & mask) * bias[k];
  }
};

// gathers of the sorted voxel arrays
struct VoxelGatherFn {
  const int32_t* xyz;
  const int32_t* order;
  int bias[3];
  int32_t* pos;
  int32_t* bpos;
  PCC_HD void operator()(int64_t i) const
  {
    const int32_t* p = &xyz[size_t(order[i]) * 3];
    for (int k = 0; k < 3; k++) {
      pos[i * 3 + k] = p[k];
      bpos[i * 3 + k] = p[k] * bias[k];
    }
  }
};

struct IotaFn {
  uint32_t* out;
  PCC_HD void operator()(int64_t i) const { out[i] = uint32_t(i); }
};

}  // namespace pccb200
