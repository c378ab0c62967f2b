// recolour.cuh — attribute transfer from a source cloud to the (re)coded
// geometry: recolourColour / recolourReflectance of the reference
// (tmc3/pointset_processing.cpp:253-923, driver :925-958, call site
// tmc3/encoder.cpp:1031-1037).  The per-item bodies are host/device functors
// (the CPU unit tests run them through tests/emu's HostExec); the schedule is
// written against the executor concept of raht_pipeline.cuh.
//
// The reference searches its neighbours with nanoflann kd-trees
// (dependencies/nanoflann; the one place in the attribute path that does).
// Here both searches are exact k-nearest-neighbour queries over a grid hash:
// the indexed points are sorted by the Morton code of their cell, a cell's
// points are one contiguous range found by binary search, and a query walks
// the cells around it ring by ring until no unvisited cell can hold a closer
// point.  Distances are the reference's (double, squared Euclidean, summed in
// axis order, no fused multiply-add); ties are broken by the lower point
// index, which nanoflann does not promise -- see DESIGN.md for what that
// means for parity (bit-exact against the oracle, which restates the same
// rule; within a stated tolerance of the compiled reference on clouds where
// distance ties reach the k-th neighbour).  The second path (kRecolourRefExact)
// searches nanoflann's own tree instead (kdtree.cuh) and orders the backward
// lists as std::sort does: equal to the reference bit for bit.
#pragma once

#include <math.h>

#include "kdtree.cuh"    // dmul / dadd / dsub, the reference-exact search
#include "raht_core.cuh"
#include "spherical.cuh"  // atomic_min_i32 / atomic_max_i32

namespace pccb200 {

constexpr int kRecolourMaxK = 16;      // neighbours per query (reference default: 8 / 1)
constexpr int kRecolourMaxRing = 24;   // rings walked before a query scans everything

struct RecolourConfig {
  double distOffsetFwd, distOffsetBwd;
  double maxGeomFwd, maxGeomBwd;   // already mapped: >= 512 -> DBL_MAX
  double maxAttrFwd, maxAttrBwd;
  int searchRange;
  int kFwd, kBwd;
  int weightedFwd, weightedBwd;
  int skipFwd, skipBwd;
  double scale;      // sourceToTargetScaleFactor
  double invScale;   // 1.0 / scale
  int off[3];        // targetToSourceOffset
  int nSrc, nTgt;
};

// One attribute set recoloured on the positions of a RecolourConfig: the
// source values (nSrc x A), the forward colours (nTgt x A, executor memory,
// filled by recolour_run) and the result (nTgt x A).
constexpr int kRecolourMaxSets = PCCB200_MAX_RECOLOUR_SETS;
struct RecolourSet {
  const int32_t* srcAttr;
  int A;          // 1 or 3
  int bitdepth;   // values are clipped to [0, (1 << bitdepth) - 1]
  int32_t* refined1;
  int32_t* out;
};

PCC_HD int
atomic_fetch_add_i32(int* p, int v)
{
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  int old = *p;
  *p += v;
  return old;
#endif
}

//----------------------------------------------------------------------------
// the grid hash over one point set

struct PointGrid {
  const int64_t* code;   // Morton code of the point's cell, ascending
  const int32_t* order;  // original index of sorted entry i
  const int32_t* spos;   // positions in sorted order (n x 3)
  int n;
  int shift;             // cell edge = 1 << shift
  const int32_t* bbox;   // [6]: min / max cell coordinate per axis
};

// cell coordinates of every point (input of the Morton sort)
struct CellCoordFn {
  const int32_t* xyz;
  int shift;
  int32_t* cell;   // n x 3
  int* flag;       // bit 0: a coordinate is negative or too large for a 63-bit Morton code
  PCC_HD void operator()(int64_t i) const
  {
    for (int k = 0; k < 3; k++) {
      const int32_t v = xyz[3 * i + k];
      if (v < 0 || v >= (1 << 21))
        atomic_or_i32(flag, 1);
      cell[3 * i + k] = v < 0 ? 0 : v >> shift;
    }
  }
};

struct GatherPosFn {
  const int32_t* xyz;
  const int32_t* order;
  int shift;
  int32_t* spos;
  int32_t* bbox;   // [6], initialised to INT_MAX x3, INT_MIN x3
  PCC_HD void operator()(int64_t i) const
  {
    const int32_t o = order[i];
    for (int k = 0; k < 3; k++) {
      const int32_t v = xyz[3 * size_t(o) + k];
      spos[3 * i + k] = v;
#if defined(__CUDA_ARCH__)
      // one atomic per warp and bound instead of one per point
      const unsigned act = __activemask();
      const int lo = __reduce_min_sync(act, v >> shift);
      const int hi = __reduce_max_sync(act, v >> shift);
      if ((threadIdx.x & 31) == __ffs(act) - 1) {
        atomicMin(&bbox[k], lo);
        atomicMax(&bbox[3 + k], hi);
      }
#else
      atomic_min_i32(&bbox[k], v >> shift);
      atomic_max_i32(&bbox[3 + k], v >> shift);
#endif
    }
  }
};

// number of distinct cells (adjacent-difference count over the sorted codes)
struct DistinctCodeFn {
  const int64_t* code;
  int* count;
  PCC_HD void operator()(int64_t i) const
  {
    const bool head = i == 0 || code[i] != code[i - 1];
#if defined(__CUDA_ARCH__)
    const unsigned act = __activemask();
    const unsigned heads = __ballot_sync(act, head);
    if (heads && (threadIdx.x & 31) == __ffs(act) - 1)
      atomicAdd(count, __popc(heads));
#else
    if (head)
      atomic_add_i32(count, 1);
#endif
  }
};

// the (dist, index)-ordered result list of one query
struct KnnList {
  double d[kRecolourMaxK];
  int32_t id[kRecolourMaxK];
  int cnt;
  int k;
  PCC_HD void insert(double dist, int32_t idx)
  {
    if (cnt == k) {
      const double w = d[k - 1];
      if (!(dist < w || (dist == w && idx < id[k - 1])))
        return;
    }
    int pos = cnt < k ? cnt : k - 1;
    while (pos > 0 && (d[pos - 1] > dist || (d[pos - 1] == dist && id[pos - 1] > idx))) {
      d[pos] = d[pos - 1];
      id[pos] = id[pos - 1];
      pos--;
    }
    d[pos] = dist;
    id[pos] = idx;
    if (cnt < k)
      cnt++;
  }
};

// squared distance as nanoflann's L2_Simple_Adaptor accumulates it
PCC_HD double
sqr_dist3(const double q[3], const int32_t* p)
{
  double r = 0.0;
  for (int k = 0; k < 3; k++) {
    const double diff = dsub(q[k], double(p[k]));
    r = dadd(r, dmul(diff, diff));
  }
  return r;
}

PCC_HD void
grid_knn(const PointGrid& g, const double q[3], KnnList& L)
{
  L.cnt = 0;
  int64_t qc[3];
  for (int k = 0; k < 3; k++)
    qc[k] = int64_t(floor(q[k])) >> g.shift;
  // the first ring that can touch the occupied box, the last one that has to
  int64_t r0 = 0, r1 = 0;
  for (int k = 0; k < 3; k++) {
    const int64_t lo = g.bbox[k], hi = g.bbox[3 + k];
    const int64_t below = lo - qc[k], above = qc[k] - hi;
    const int64_t gap = below > 0 ? below : above > 0 ? above : 0;
    r0 = gap > r0 ? gap : r0;
    const int64_t a = qc[k] - lo, b = hi - qc[k];
    const int64_t far = (a > b ? a : b);
    r1 = far > r1 ? far : r1;
  }
  const double cs = double(int64_t(1) << g.shift);
  bool scanAll = false;
  for (int64_t r = r0; r <= r1; r++) {
    if (r - r0 > kRecolourMaxRing) {
      scanAll = true;
      break;
    }
    for (int64_t dz = -r; dz <= r; dz++) {
      const int64_t cz = qc[2] + dz;
      if (cz < g.bbox[2] || cz > g.bbox[5])
        continue;
      for (int64_t dy = -r; dy <= r; dy++) {
        const int64_t cy = qc[1] + dy;
        if (cy < g.bbox[1] || cy > g.bbox[4])
          continue;
        const bool shell = dz == -r || dz == r || dy == -r || dy == r;
        // inside the shell's faces only the two end cells of the row belong to ring r
        for (int64_t dx = -r; dx <= r; dx += (shell || r == 0) ? 1 : 2 * r) {
          const int64_t cx = qc[0] + dx;
          if (cx < g.bbox[0] || cx > g.bbox[3])
            continue;
          const int64_t cell = morton_addr(int32_t(cx), int32_t(cy), int32_t(cz));
          int a = 0, b = g.n;
          while (a < b) {
            const int m = (a + b) >> 1;
            if (g.code[m] < cell)
              a = m + 1;
            else
              b = m;
          }
          for (int i = a; i < g.n && g.code[i] == cell; i++)
            L.insert(sqr_dist3(q, &g.spos[3 * size_t(i)]), g.order[i]);
        }
      }
    }
    // every unvisited point is farther than r cells along some axis
    if (L.cnt == L.k) {
      const double bound = dmul(double(r) * cs, double(r) * cs);
      if (L.d[L.k - 1] <= bound)
        return;
    }
  }
  if (scanAll) {
    L.cnt = 0;
    for (int i = 0; i < g.n; i++)
      L.insert(sqr_dist3(q, &g.spos[3 * size_t(i)]), g.order[i]);
  }
}

// one query per item: the target points in the source (forward,
// pointset_processing.cpp:306-313) or the source points in the target
// (backward, :409-418)
struct KnnQueryFn {
  PointGrid g;
  RecolourConfig cfg;
  const int32_t* qxyz;
  int backward;
  int k;
  double* outDist;    // nQueries x k
  int32_t* outIdx;
  PCC_HD void operator()(int64_t i) const
  {
    double q[3];
    for (int c = 0; c < 3; c++) {
      if (backward)  // posInTgt = source * scale - offset
        q[c] = dsub(dmul(double(qxyz[3 * i + c]), cfg.scale), double(cfg.off[c]));
      else  // posInSrc = (target + offset) * (1 / scale)
        q[c] = dmul(double(qxyz[3 * i + c] + cfg.off[c]), cfg.invScale);
    }
    KnnList L;
    L.k = k;
    grid_knn(g, q, L);
    for (int j = 0; j < k; j++) {
      outDist[size_t(i) * k + j] = j < L.cnt ? L.d[j] : 0.0;
      outIdx[size_t(i) * k + j] = j < L.cnt ? L.id[j] : -1;
    }
  }
};

// the same queries through nanoflann's tree and search (kdtree.cuh)
struct KdKnnQueryFn {
  KdTree T;
  RecolourConfig cfg;
  const int32_t* qxyz;
  int backward;
  int k;
  double* outDist;    // nQueries x k
  int32_t* outIdx;
  PCC_HD void operator()(int64_t i) const
  {
    double q[3];
    for (int c = 0; c < 3; c++) {
      if (backward)
        q[c] = dsub(dmul(double(qxyz[3 * i + c]), cfg.scale), double(cfg.off[c]));
      else
        q[c] = dmul(double(qxyz[3 * i + c] + cfg.off[c]), cfg.invScale);
    }
    KdResult R;
    R.init(k);
    kd_find_neighbours(T, q, R);
    for (int j = 0; j < k; j++) {
      outDist[size_t(i) * k + j] = j < R.count ? R.d[j] : 0.0;
      outIdx[size_t(i) * k + j] = j < R.count ? R.id[j] : -1;
    }
  }
};

// The reference pops its result vectors when the k-th neighbour is farther
// than maxGeometryDist2Fwd -- and never restores them (the vectors live
// outside the loop, pointset_processing.cpp:301-326): from the first such
// target on, every target sees one neighbour.  firstBad = that target.
struct FirstBadFn {
  const double* dist;
  int k;
  double maxGeom;
  int32_t* firstBad;
  PCC_HD void operator()(int64_t i) const
  {
    if (k > 1 && dist[size_t(i) * k + (k - 1)] > maxGeom)
      atomic_min_i32(firstBad, int32_t(i));
  }
};

PCC_HD double
clip_round(double v, double hi)
{
  const double r = round(v);
  return r < 0.0 ? 0.0 : r > hi ? hi : r;
}

// forward colour of every target (pointset_processing.cpp:301-399 / :660-744):
// one thread per target, its neighbour list read once for every set.
// kRefExact: the attribute distance of a colour is taken as the reference
// takes it, on Vec3<attr_t> differences (:337-348), each component wrapped to
// uint16 before it is squared; a reflectance difference is a plain int (:709).
template<bool kRefExact>
struct ForwardColourT {
  RecolourConfig cfg;
  const double* dist;     // nTgt x kFwd
  const int32_t* idx;
  const int32_t* firstBad;
  int numSets;
  RecolourSet sets[kRecolourMaxSets];
  PCC_HD void operator()(int64_t t) const
  {
    const int k = cfg.kFwd;
    const double* d = dist + size_t(t) * k;
    const int32_t* id = idx + size_t(t) * k;
    int nNN0 = t >= *firstBad ? 1 : k;
    if (cfg.skipFwd && d[0] < 0.0001)
      nNN0 = 1;
    for (int si = 0; si < numSets; si++) {
      const RecolourSet& S = sets[si];
      const int A = S.A;
      const int32_t* srcAttr = S.srcAttr;
      const double clipMax = double((1 << S.bitdepth) - 1);
      int32_t* refined1 = S.refined1 + size_t(t) * A;
      int nNN = nNN0;
      while (nNN > 1) {
        double maxAttr = 2.2250738585072014e-308;  // std::numeric_limits<double>::min()
        for (int i = 0; i < nNN; i++)
          for (int j = 0; j < nNN; j++) {
            double s = 0.0;
            for (int c = 0; c < A; c++) {
              double df = double(srcAttr[size_t(id[i]) * A + c])
                - double(srcAttr[size_t(id[j]) * A + c]);
              if constexpr (kRefExact) {
                if (A == 3)
                  df = double(uint16_t(srcAttr[size_t(id[i]) * A + c] - srcAttr[size_t(id[j]) * A + c]));
              }
              s = dadd(s, dmul(df, df));
            }
            if (s > maxAttr)
              maxAttr = s;
          }
        if (maxAttr > cfg.maxAttrFwd) {
          --nNN;
          continue;
        }
        double acc[3] = {0.0, 0.0, 0.0};
        if (cfg.weightedFwd) {
          double sumW = 0.0;
          for (int i = 0; i < nNN; i++) {
            const double w = 1 / dadd(d[i], cfg.distOffsetFwd);
            for (int c = 0; c < A; c++)
              acc[c] = dadd(acc[c], dmul(double(srcAttr[size_t(id[i]) * A + c]), w));
            sumW = dadd(sumW, w);
          }
          for (int c = 0; c < A; c++)
            acc[c] = acc[c] / sumW;
        } else {
          for (int i = 0; i < nNN; i++)
            for (int c = 0; c < A; c++)
              acc[c] = dadd(acc[c], double(srcAttr[size_t(id[i]) * A + c]));
          for (int c = 0; c < A; c++)
            acc[c] = acc[c] / double(nNN);
        }
        for (int c = 0; c < A; c++)
          refined1[c] = int32_t(clip_round(acc[c], clipMax));
        break;
      }
      if (nNN <= 1)
        for (int c = 0; c < A; c++)
          refined1[c] = srcAttr[size_t(id[0]) * A + c];
    }
  }
};

using ForwardColourFn = ForwardColourT<false>;

// backward lists: the sources that name a target among their kBwd nearest
// (pointset_processing.cpp:409-428), as CSR: count, (scan), fill, sort.
struct BackwardCountFn {
  RecolourConfig cfg;
  const double* dist;   // nSrc x kBwd
  const int32_t* idx;
  int* count;           // nTgt (+1)
  PCC_HD void operator()(int64_t s) const
  {
    for (int j = 0; j < cfg.kBwd; j++) {
      const int32_t t = idx[size_t(s) * cfg.kBwd + j];
      if (t >= 0 && dist[size_t(s) * cfg.kBwd + j] <= cfg.maxGeomBwd)
        atomic_add_i32(&count[t], 1);
    }
  }
};

struct BackwardFillFn {
  RecolourConfig cfg;
  const double* dist;
  const int32_t* idx;
  const int* first;     // nTgt + 1 (exclusive scan of the counts)
  int* cursor;          // nTgt, zeroed
  double* listDist;
  int32_t* listSrc;
  PCC_HD void operator()(int64_t s) const
  {
    for (int j = 0; j < cfg.kBwd; j++) {
      const int32_t t = idx[size_t(s) * cfg.kBwd + j];
      const double d = dist[size_t(s) * cfg.kBwd + j];
      if (t >= 0 && d <= cfg.maxGeomBwd) {
        const int at = first[t] + atomic_fetch_add_i32(&cursor[t], 1);
        listDist[at] = d;
        listSrc[at] = int32_t(s);
      }
    }
  }
};

// final colour of every target (pointset_processing.cpp:430-611 / :773-921):
// one thread per target sorts its backward list once, then runs the centroid
// and the search of every set.  kRefOrder = false: the list is ordered by
// (dist, source index).  kRefOrder = true: in the order the reference's
// std::sort on distance leaves it -- the list as it was pushed (by source
// index), then libstdc++'s introsort (GnuSort) keyed on distance alone.
template<bool kRefOrder>
struct FinalColourT {
  RecolourConfig cfg;
  const int* first;
  double* listDist;     // sorted in place (see kRefOrder)
  int32_t* listSrc;
  int numSets;
  RecolourSet sets[kRecolourMaxSets];
  PCC_HD void operator()(int64_t t) const
  {
    const int lo = first[t];
    const int L0 = first[t + 1] - lo;
    double* ld = listDist + lo;
    int32_t* ls = listSrc + lo;
    if (L0 == 0) {
      for (int si = 0; si < numSets; si++)
        for (int c = 0; c < sets[si].A; c++)
          sets[si].out[size_t(t) * sets[si].A + c] = sets[si].refined1[size_t(t) * sets[si].A + c];
      return;
    }
    if constexpr (kRefOrder) {
      GnuSort<int32_t, double, IndexLess>{ls, ld, IndexLess{}}(L0);
      GnuSort<double, int32_t, DistLess>{ld, ls, DistLess{}}(L0);
    } else {
      // std::sort by distance (the reference's order among equal distances is
      // unspecified; here: by source index)
      for (int i = 1; i < L0; i++) {
        const double d = ld[i];
        const int32_t s = ls[i];
        int p = i;
        while (p > 0 && (ld[p - 1] > d || (ld[p - 1] == d && ls[p - 1] > s))) {
          ld[p] = ld[p - 1];
          ls[p] = ls[p - 1];
          p--;
        }
        ld[p] = d;
        ls[p] = s;
      }
    }
    for (int si = 0; si < numSets; si++) {
      const RecolourSet& S = sets[si];
      const int A = S.A;
      const int32_t* srcAttr = S.srcAttr;
      const double clipMax = double((1 << S.bitdepth) - 1);
      const int32_t* c1 = S.refined1 + size_t(t) * A;
      int L = L0;
      double centroid2[3] = {0.0, 0.0, 0.0};
      bool done = false;
      if (cfg.skipBwd && ld[0] < 0.0001) {
        L = 1;
        done = true;
      }
      while (!done) {
        if (L == 1) {
          done = true;
          break;
        }
        double maxAttr = 2.2250738585072014e-308;
        for (int i = 0; i < L; i++)
          for (int j = 0; j < L; j++) {
            double s = 0.0;
            for (int c = 0; c < A; c++) {
              const double df = double(srcAttr[size_t(ls[i]) * A + c])
                - double(srcAttr[size_t(ls[j]) * A + c]);
              s = dadd(s, dmul(df, df));
            }
            if (s > maxAttr)
              maxAttr = s;
          }
        if (maxAttr <= cfg.maxAttrBwd) {
          if (cfg.weightedBwd) {
            double sumW = 0.0;
            for (int i = 0; i < L; i++) {
              const double w = 1 / dadd(sqrt(ld[i]), cfg.distOffsetBwd);
              for (int c = 0; c < A; c++)
                centroid2[c] = dadd(centroid2[c], dmul(double(srcAttr[size_t(ls[i]) * A + c]), w));
              sumW = dadd(sumW, w);
            }
            for (int c = 0; c < A; c++)
              centroid2[c] = centroid2[c] / sumW;
          } else {
            for (int i = 0; i < L; i++)
              for (int c = 0; c < A; c++)
                centroid2[c] = dadd(centroid2[c], double(srcAttr[size_t(ls[i]) * A + c]));
            for (int c = 0; c < A; c++)
              centroid2[c] = centroid2[c] / double(L);
          }
          break;
        }
        L--;  // pop_back
      }
      if (done)
        for (int c = 0; c < A; c++)
          centroid2[c] = double(srcAttr[size_t(ls[0]) * A + c]);
      // fixWeight (m42538): w = 0, the starting point is centroid2
      double c0[3] = {0.0, 0.0, 0.0};
      for (int c = 0; c < A; c++)
        c0[c] = clip_round(dadd(dmul(0.0, double(c1[c])), dmul(1.0, centroid2[c])), clipMax);
      const double rSource = 1.0 / double(cfg.nSrc);
      const double rTarget = 1.0 / double(cfg.nTgt);
      double minError = 1.7976931348623157e308;
      double best[3] = {c0[0], c0[1], c0[2]};
      const int R = cfg.searchRange;
      const int R1 = A == 3 ? R : 0;  // the single-component search is one loop
      double col[3] = {0.0, 0.0, 0.0};
      for (int s1 = -R; s1 <= R; s1++) {
        col[0] = c0[0] + s1 < 0.0 ? 0.0 : c0[0] + s1 > clipMax ? clipMax : c0[0] + s1;
        for (int s2 = -R1; s2 <= R1; s2++) {
          if (A == 3)
            col[1] = c0[1] + s2 < 0.0 ? 0.0 : c0[1] + s2 > clipMax ? clipMax : c0[1] + s2;
          for (int s3 = -R1; s3 <= R1; s3++) {
            if (A == 3)
              col[2] = c0[2] + s3 < 0.0 ? 0.0 : c0[2] + s3 > clipMax ? clipMax : c0[2] + s3;
            double e1 = 0.0;
            for (int c = 0; c < A; c++) {
              const double df = dsub(col[c], double(c1[c]));
              e1 = dadd(e1, dmul(df, df));
            }
            e1 = dmul(e1, rTarget);
            double e2 = 0.0;
            for (int i = 0; i < L; i++)
              for (int c = 0; c < A; c++) {
                const double df = dsub(col[c], double(srcAttr[size_t(ls[i]) * A + c]));
                e2 = dadd(e2, dmul(df, df));
              }
            e2 = dmul(e2, rSource);
            const double err = e1 > e2 ? e1 : e2;
            if (err < minError) {
              minError = err;
              for (int c = 0; c < A; c++)
                best[c] = col[c];
            }
          }
        }
      }
      int32_t* out = S.out + size_t(t) * A;
      for (int c = 0; c < A; c++)
        out[c] = int32_t(best[c]);
    }
  }
};

using FinalColourFn = FinalColourT<false>;

struct FillI32ValueFn {
  int32_t* p;
  int32_t v;
  PCC_HD void operator()(int64_t i) const { p[i] = v; }
};

//----------------------------------------------------------------------------
// schedule

// builds the grid over n points (executor memory); the cell size is the
// smallest power of two that leaves at most n / 2 occupied cells (about two or
// more points per occupied cell), found by trying shifts (each try is one sort)
template<class Exec>
int
build_point_grid(Exec& ex, const int32_t* xyz, int n, PointGrid& g)
{
  int32_t* cell = ex.template alloc<int32_t>(size_t(n) * 3);
  int64_t* code = ex.template alloc<int64_t>(n);
  int32_t* order = ex.template alloc<int32_t>(n);
  int* flag = ex.template alloc<int>(2);
  int shift = 0;
  for (;; shift++) {
    ex.zero(flag, 2 * sizeof(int));
    ex.foreach(n, CellCoordFn{xyz, shift, cell, flag});
    ex.morton_sort(cell, n, code, order);
    ex.foreach(n, DistinctCodeFn{code, flag + 1});
    int h[2];
    ex.download(h, flag, sizeof(h));
    if (h[0] & 1)
      return PCCB200_ERR_INVALID_ARG;
    if (h[1] <= (n + 1) / 2 || shift >= 20)
      break;
  }
  int32_t* spos = ex.template alloc<int32_t>(size_t(n) * 3);
  int32_t* bbox = ex.template alloc<int32_t>(6);
  const int32_t init[6] = {INT32_MAX, INT32_MAX, INT32_MAX, INT32_MIN, INT32_MIN, INT32_MIN};
  ex.upload(bbox, init, sizeof(init));
  ex.foreach(n, GatherPosFn{xyz, order, shift, spos, bbox});
  g.code = code;
  g.order = order;
  g.spos = spos;
  g.n = n;
  g.shift = shift;
  g.bbox = bbox;
  return PCCB200_OK;
}

// The arguments recolour_run accepts: at least one point on each side, 1 to
// kRecolourMaxSets sets of 1 or 3 components at 1 to 16 bits, neighbour counts
// within kRecolourMaxK and the point counts, a search range of 0 to 8 and a
// positive scale.  (Coordinates outside [0, 2^21) are found by build_point_grid,
// those outside (-2^30, 2^30) of the reference-exact search by kd_coords_valid.)
inline bool
recolour_args_valid(const pccb200_recolour_params& rp, int nSrc, int nTgt, double scale,
                    int numSets, const RecolourSet* sets)
{
  if (nSrc <= 0 || nTgt <= 0 || numSets < 1 || numSets > kRecolourMaxSets
      || rp.num_neighbours_fwd < 1 || rp.num_neighbours_fwd > kRecolourMaxK
      || rp.num_neighbours_bwd < 1 || rp.num_neighbours_bwd > kRecolourMaxK
      || rp.num_neighbours_fwd > nSrc || rp.num_neighbours_bwd > nTgt || rp.search_range < 0
      || rp.search_range > 8 || !(scale > 0.0))
    return false;
  for (int s = 0; s < numSets; s++)
    if ((sets[s].A != 1 && sets[s].A != 3) || sets[s].bitdepth < 1 || sets[s].bitdepth > 16)
      return false;
  return true;
}

// The neighbour search and backward-list order of a recolour_run call.
//   kRecolourGrid: exact k nearest over grid hashes, ties by the lower point
//     index, lists by (dist, source index); coordinates in [0, 2^21).
//   kRecolourRefExact: nanoflann's trees and traversal (kdtree.cuh), lists in
//     libstdc++'s std::sort order: the reference's recolourColour /
//     recolourReflectance bit for bit; coordinates (and offsets) of |x| < 2^30.
enum RecolourSearch { kRecolourGrid = 0, kRecolourRefExact = 1 };

// |x| < 2^30 for every coordinate of both sides and the offset
template<class Exec>
bool
kd_coords_valid(Exec& ex, const int32_t* srcXyz, int nSrc, const int32_t* tgtXyz, int nTgt,
                const int32_t off[3])
{
  for (int k = 0; k < 3; k++)
    if (off[k] <= -(1 << 30) || off[k] >= (1 << 30))
      return false;
  int* flag = ex.template alloc<int>(1);
  ex.zero(flag, sizeof(int));
  ex.foreach(nSrc, KdCoordCheckFn{srcXyz, flag});
  ex.foreach(nTgt, KdCoordCheckFn{tgtXyz, flag});
  int h = 0;
  ex.download(&h, flag, sizeof(int));
  return h == 0;
}

// Recolours numSets attribute sets on the same source and target positions.
// The grids (or trees), both neighbour searches and the backward lists are
// built once; the forward and final colours of all sets are computed by one
// launch each, so the launches do not depend on numSets.  sets[s]: srcAttr, A,
// bitdepth and out (srcXyz / tgtXyz / srcAttr / out: executor memory);
// refined1 is allocated here.  Returns a PCCB200_* status.
template<class Exec>
int
recolour_run(Exec& ex, const pccb200_recolour_params& rp, const int32_t* srcXyz, int nSrc,
             double sourceToTargetScale, const int32_t off[3], const int32_t* tgtXyz, int nTgt,
             int numSets, const RecolourSet* sets, RecolourSearch search = kRecolourGrid)
{
  if (!recolour_args_valid(rp, nSrc, nTgt, sourceToTargetScale, numSets, sets))
    return PCCB200_ERR_INVALID_ARG;
  const bool exact = search == kRecolourRefExact;
  RecolourConfig cfg;
  const double big = 1.7976931348623157e308;
  cfg.distOffsetFwd = rp.dist_offset_fwd;
  cfg.distOffsetBwd = rp.dist_offset_bwd;
  cfg.maxGeomFwd = rp.max_geometry_dist2_fwd < 512 ? rp.max_geometry_dist2_fwd : big;
  cfg.maxGeomBwd = rp.max_geometry_dist2_bwd < 512 ? rp.max_geometry_dist2_bwd : big;
  cfg.maxAttrFwd = rp.max_attribute_dist2_fwd < 512 ? rp.max_attribute_dist2_fwd : big;
  cfg.maxAttrBwd = rp.max_attribute_dist2_bwd < 512 ? rp.max_attribute_dist2_bwd : big;
  cfg.searchRange = rp.search_range;
  cfg.kFwd = rp.num_neighbours_fwd;
  cfg.kBwd = rp.num_neighbours_bwd;
  cfg.weightedFwd = rp.use_dist_weighted_avg_fwd != 0;
  cfg.weightedBwd = rp.use_dist_weighted_avg_bwd != 0;
  cfg.skipFwd = rp.skip_avg_if_identical_source_point_present_fwd != 0;
  cfg.skipBwd = rp.skip_avg_if_identical_source_point_present_bwd != 0;
  cfg.scale = sourceToTargetScale;
  cfg.invScale = 1.0 / sourceToTargetScale;
  for (int k = 0; k < 3; k++)
    cfg.off[k] = off[k];
  cfg.nSrc = nSrc;
  cfg.nTgt = nTgt;

  ex.phase(0);
  PointGrid gs, gt;
  KdTree ts, tt;
  int rc;
  if (exact) {
    if (!kd_coords_valid(ex, srcXyz, nSrc, tgtXyz, nTgt, off))
      return PCCB200_ERR_INVALID_ARG;
    rc = build_kdtree(ex, srcXyz, nSrc, ts);
    if (rc == PCCB200_OK)
      rc = build_kdtree(ex, tgtXyz, nTgt, tt);
  } else {
    rc = build_point_grid(ex, srcXyz, nSrc, gs);
    if (rc == PCCB200_OK)
      rc = build_point_grid(ex, tgtXyz, nTgt, gt);
  }
  if (rc != PCCB200_OK)
    return rc;

  //-- forward: every target in the source
  ex.phase(2);
  double* fDist = ex.template alloc<double>(size_t(nTgt) * cfg.kFwd);
  int32_t* fIdx = ex.template alloc<int32_t>(size_t(nTgt) * cfg.kFwd);
  if (exact)
    ex.foreach(nTgt, KdKnnQueryFn{ts, cfg, tgtXyz, 0, cfg.kFwd, fDist, fIdx});
  else
    ex.foreach(nTgt, KnnQueryFn{gs, cfg, tgtXyz, 0, cfg.kFwd, fDist, fIdx});
  int32_t* firstBad = ex.template alloc<int32_t>(1);
  const int32_t never = INT32_MAX;
  ex.upload(firstBad, &never, sizeof(never));
  ex.foreach(nTgt, FirstBadFn{fDist, cfg.kFwd, cfg.maxGeomFwd, firstBad});
  RecolourSet withRefined[kRecolourMaxSets];
  for (int s = 0; s < numSets; s++) {
    withRefined[s] = sets[s];
    withRefined[s].refined1 = ex.template alloc<int32_t>(size_t(nTgt) * sets[s].A);
  }
  if (exact) {
    ForwardColourT<true> fwd{cfg, fDist, fIdx, firstBad, numSets, {}};
    for (int s = 0; s < numSets; s++)
      fwd.sets[s] = withRefined[s];
    ex.foreach(nTgt, fwd);
  } else {
    ForwardColourFn fwd{cfg, fDist, fIdx, firstBad, numSets, {}};
    for (int s = 0; s < numSets; s++)
      fwd.sets[s] = withRefined[s];
    ex.foreach(nTgt, fwd);
  }

  //-- backward: every source in the target, lists per target
  double* bDist = ex.template alloc<double>(size_t(nSrc) * cfg.kBwd);
  int32_t* bIdx = ex.template alloc<int32_t>(size_t(nSrc) * cfg.kBwd);
  if (exact)
    ex.foreach(nSrc, KdKnnQueryFn{tt, cfg, srcXyz, 1, cfg.kBwd, bDist, bIdx});
  else
    ex.foreach(nSrc, KnnQueryFn{gt, cfg, srcXyz, 1, cfg.kBwd, bDist, bIdx});
  int* first = ex.template alloc<int>(size_t(nTgt) + 1);
  ex.zero(first, (size_t(nTgt) + 1) * sizeof(int));
  ex.foreach(nSrc, BackwardCountFn{cfg, bDist, bIdx, first});
  ex.exclusive_scan(first, int64_t(nTgt) + 1);
  int* cursor = ex.template alloc<int>(nTgt);
  ex.zero(cursor, size_t(nTgt) * sizeof(int));
  const size_t maxPairs = size_t(nSrc) * cfg.kBwd;
  double* listDist = ex.template alloc<double>(maxPairs);
  int32_t* listSrc = ex.template alloc<int32_t>(maxPairs);
  ex.foreach(nSrc, BackwardFillFn{cfg, bDist, bIdx, first, cursor, listDist, listSrc});

  //-- the colour of every target, every set
  ex.phase(3);
  if (exact) {
    FinalColourT<true> fin{cfg, first, listDist, listSrc, numSets, {}};
    for (int s = 0; s < numSets; s++)
      fin.sets[s] = withRefined[s];
    ex.foreach(nTgt, fin);
  } else {
    FinalColourFn fin{cfg, first, listDist, listSrc, numSets, {}};
    for (int s = 0; s < numSets; s++)
      fin.sets[s] = withRefined[s];
    ex.foreach(nTgt, fin);
  }
  return PCCB200_OK;
}

// one attribute set (srcAttr: nSrc x A, out: nTgt x A)
template<class Exec>
int
recolour_run(Exec& ex, const pccb200_recolour_params& rp, const int32_t* srcXyz,
             const int32_t* srcAttr, int A, int nSrc, double sourceToTargetScale,
             const int32_t off[3], const int32_t* tgtXyz, int nTgt, int bitdepth, int32_t* out,
             RecolourSearch search = kRecolourGrid)
{
  const RecolourSet set{srcAttr, A, bitdepth, nullptr, out};
  return recolour_run(ex, rp, srcXyz, nSrc, sourceToTargetScale, off, tgtXyz, nTgt, 1, &set,
                      search);
}

}  // namespace pccb200
