// kdtree.cuh — the reference's k-nearest-neighbour search, reproduced: the
// tree nanoflann builds for KDTreeVectorOfVectorsAdaptor<PCCPointSet3, double>
// (metric_L2, leaf size 10, no bounding-box hint), built on the device, and its
// findNeighbors / searchLevel with a KNNResultSet, one thread per query.  Used
// by the reference-exact recolouring (recolour.cuh, kRecolourRefExact): among
// equidistant candidates nanoflann keeps the one its traversal meets first, so
// equal results need the same tree and the same traversal, not just "the k
// nearest".  Also the order libstdc++'s std::sort leaves equal keys in
// (GnuSort), which decides the order of the reference's backward lists.
//
// Build.  nanoflann's divideTree recurses depth first; here every node of one
// level is split by the same launches.  A node's split depends only on its own
// range of the index permutation (vind) and on its loose bounding box (the
// parent's loose box with the cut value substituted), and sibling ranges are
// disjoint, so the level order produces the same tree.  Per level:
//   - the tight min / max of every node's points (atomics);
//   - per node: leaf (<= 10 points) or middleSplit_'s split dimension and value;
//   - planeSplit's two Hoare passes ("< cut" over the range, then "<= cut"
//     from lim1).  A Hoare pass swaps the i-th misplaced element from the left
//     with the i-th misplaced element from the right; an exclusive scan of the
//     "belongs left" flags gives every misplaced element its rank, so the pairs
//     are formed and swapped in parallel;
//   - per node: the split index from lim1, lim2 and count / 2, and the children.
// divlow / divhigh are the children's tight bounds along the cut dimension
// (nanoflann returns a subtree's tight box from divideTree).  The tight box of
// a subtree is the min / max of its points, which the children's own level
// computes anyway, so each child writes its parent's bound there.
//
// All comparisons and products are in double without contraction (dmul /
// dadd / dsub), as the reference is compiled.
#pragma once

#include <float.h>

#include "raht_core.cuh"
#include "spherical.cuh"  // atomic_min_i32 / atomic_max_i32

namespace pccb200 {

constexpr int kKdLeafSize = 10;  // KDTreeVectorOfVectorsAdaptor's leaf_max_size
// The deepest leaf: every split leaves each child with at most half the points
// of its parent or with half its parent's loose span along the cut dimension
// while its points still spread along it; with fewer than 2^31 points and
// coordinates of |x| < 2^30 that is at most 31 + 3 * 31 levels below the root.
constexpr int kKdMaxDepth = 128;
constexpr int kKdResultMax = 16;  // neighbours per query

// exact products and sums (the compiler must not contract them into FMAs:
// the reference is built without)
PCC_HD double
dmul(double a, double b)
{
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
PCC_HD double
dadd(double a, double b)
{
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
PCC_HD double
dsub(double a, double b)
{
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// The tree as the search reads it.  Node 0 is the root; an internal node's
// children are nodes child[i] and child[i] + 1 (nanoflann's child1 / child2).
struct KdTree {
  const int32_t* vind;   // n: point index at tree position i
  const int32_t* tpos;   // n x 3: the points in tree order
  const int32_t* child;  // per node: first child, -1 for a leaf
  const int32_t* lo;     // per node: tree positions [lo, hi)
  const int32_t* hi;
  const int32_t* feat;   // divfeat (-1 for a leaf)
  const double* divLow;
  const double* divHigh;
  double rootLow[3], rootHigh[3];  // root_bbox
  int n;
  int numNodes;
  int depth;             // of the deepest leaf (root: 0)
};

// the build's per-node working state (executor memory, 2n - 1 nodes at most)
struct KdBuild {
  int32_t* lo;
  int32_t* hi;
  int32_t* child;
  int32_t* feat;
  int32_t* parent;
  int32_t* index;    // split index (children: [lo, lo + index), [lo + index, hi))
  double* divLow;
  double* divHigh;
  double* cut;
  double* box;       // 6 per node: loose low x3, high x3
  int32_t* mn;       // 3 per node: tight min / max
  int32_t* mx;
};

// vind = identity, every point in the root
struct KdInitFn {
  int32_t* vind;
  int32_t* seg;
  PCC_HD void operator()(int64_t i) const
  {
    vind[i] = int32_t(i);
    seg[i] = 0;
  }
};

// |x| < 2^30 for every coordinate (a query adds an offset of the same bound)
struct KdCoordCheckFn {
  const int32_t* xyz;
  int* flag;
  PCC_HD void operator()(int64_t i) const
  {
    for (int k = 0; k < 3; k++) {
      const int32_t v = xyz[3 * i + k];
      if (v <= -(1 << 30) || v >= (1 << 30))
        atomic_or_i32(flag, 1);
    }
  }
};

struct KdNodeInitFn {
  KdBuild B;
  int base;
  PCC_HD void operator()(int64_t j) const
  {
    const int64_t i = base + j;
    for (int k = 0; k < 3; k++) {
      B.mn[3 * i + k] = INT32_MAX;
      B.mx[3 * i + k] = INT32_MIN;
    }
  }
};

// tight min / max of every active node (seg[p]: the node of tree position p,
// -1 once its leaf is made)
struct KdMinMaxFn {
  KdBuild B;
  const int32_t* xyz;
  const int32_t* vind;
  const int32_t* seg;
  PCC_HD void operator()(int64_t p) const
  {
    const int32_t s = seg[p];
    if (s < 0)
      return;
    const int32_t* v = xyz + 3 * size_t(vind[p]);
#if defined(__CUDA_ARCH__)
    // a node's points are contiguous: most warps update one node only
    const unsigned act = __activemask();
    if (__match_any_sync(act, s) == act) {
      const bool leader = (threadIdx.x & 31) == __ffs(act) - 1;
      for (int k = 0; k < 3; k++) {
        const int lo = __reduce_min_sync(act, v[k]);
        const int hi = __reduce_max_sync(act, v[k]);
        if (leader) {
          atomicMin(&B.mn[3 * size_t(s) + k], lo);
          atomicMax(&B.mx[3 * size_t(s) + k], hi);
        }
      }
      return;
    }
#endif
    for (int k = 0; k < 3; k++) {
      atomic_min_i32(&B.mn[3 * size_t(s) + k], v[k]);
      atomic_max_i32(&B.mx[3 * size_t(s) + k], v[k]);
    }
  }
};

// Per node of the level: its bound in the parent (divlow from the left child,
// divhigh from the right), then leaf, or middleSplit_'s dimension and value.
// split[j] = 1 if the node splits (two children on the next level).
struct KdSplitFn {
  KdBuild B;
  int base;
  int* split;
  PCC_HD void operator()(int64_t j) const
  {
    const int64_t i = base + j;
    const int32_t* mn = B.mn + 3 * i;
    const int32_t* mx = B.mx + 3 * i;
    double* box = B.box + 6 * i;
    const int32_t par = B.parent[i];
    if (par < 0) {  // root: root_bbox = computeBoundingBox
      for (int k = 0; k < 3; k++) {
        box[k] = double(mn[k]);
        box[3 + k] = double(mx[k]);
      }
    } else {
      const int f = B.feat[par];
      if (i == B.child[par])
        B.divLow[par] = double(mx[f]);
      else
        B.divHigh[par] = double(mn[f]);
    }
    if (B.hi[i] - B.lo[i] <= kKdLeafSize) {
      B.child[i] = -1;
      B.feat[i] = -1;
      split[j] = 0;
      return;
    }
    const double EPS = 0.00001;
    double span[3];
    for (int k = 0; k < 3; k++)
      span[k] = dsub(box[3 + k], box[k]);
    double maxSpan = span[0];
    for (int k = 1; k < 3; k++)
      if (span[k] > maxSpan)
        maxSpan = span[k];
    double maxSpread = -1;
    int cf = 0;
    for (int k = 0; k < 3; k++) {
      if (span[k] >= dmul(1 - EPS, maxSpan)) {
        const double spread = dsub(double(mx[k]), double(mn[k]));
        if (spread > maxSpread) {
          cf = k;
          maxSpread = spread;
        }
      }
    }
    const double splitVal = dadd(box[cf], box[3 + cf]) / 2;
    const double lo = double(mn[cf]), hi = double(mx[cf]);
    B.feat[i] = cf;
    B.cut[i] = splitVal < lo ? lo : splitVal > hi ? hi : splitVal;
    split[j] = 1;
  }
};

// One Hoare pass of planeSplit over the internal nodes of the level, in three
// launches.  Pass 0: "left" = (v < cut) over [lo, hi); pass 1: "left" =
// (v <= cut) over [lo + lim1, hi).  KdFlagFn writes the flags (n + 1 entries,
// the last 0) for an exclusive scan: the scan's difference over a range counts
// its left elements, so lim = start + scan[hi] - scan[start].
struct KdPass {
  const int32_t* xyz;
  int32_t* vind;
  const int32_t* seg;
  const int* scan0;   // pass 0's scanned flags (pass 1 reads lim1 from them)
  int pass;
  // the node of position p and its pass range start, or -1
  PCC_HD int32_t node(const KdBuild& B, int64_t p, int32_t& start) const
  {
    const int32_t s = seg[p];
    if (s < 0 || B.feat[s] < 0)
      return -1;
    start = B.lo[s];
    if (pass)
      start += scan0[B.hi[s]] - scan0[B.lo[s]];
    return p >= start ? s : -1;
  }
};

struct KdFlagFn {
  KdBuild B;
  KdPass P;
  int n;
  int* flag;
  PCC_HD void operator()(int64_t p) const
  {
    int32_t start, s = -1;
    if (p < n)
      s = P.node(B, p, start);
    int f = 0;
    if (s >= 0) {
      const double v = double(P.xyz[3 * size_t(P.vind[p]) + B.feat[s]]);
      f = P.pass ? v <= B.cut[s] : v < B.cut[s];
    }
    flag[p] = f;
  }
};

// the misplaced elements right of the boundary (left elements at or after
// start + count): the i-th from the right records its position in slot[start + i]
struct KdPairRightFn {
  KdBuild B;
  KdPass P;
  const int* scan;
  int32_t* slot;
  PCC_HD void operator()(int64_t p) const
  {
    int32_t start;
    const int32_t s = P.node(B, p, start);
    if (s < 0 || scan[p + 1] == scan[p])
      return;
    const int32_t hi = B.hi[s];
    const int32_t mid = start + (scan[hi] - scan[start]);
    if (p >= mid)
      slot[start + (scan[hi] - scan[p + 1])] = int32_t(p);
  }
};

// the misplaced elements left of the boundary: the i-th from the left swaps
// with the i-th from the right
struct KdPairLeftFn {
  KdBuild B;
  KdPass P;
  const int* scan;
  const int32_t* slot;
  PCC_HD void operator()(int64_t p) const
  {
    int32_t start;
    const int32_t s = P.node(B, p, start);
    if (s < 0 || scan[p + 1] != scan[p])
      return;
    const int32_t mid = start + (scan[B.hi[s]] - scan[start]);
    if (p >= mid)
      return;
    const int32_t rank = int32_t(p - start) - (scan[p] - scan[start]);
    const int32_t q = slot[start + rank];
    const int32_t t = P.vind[p];
    P.vind[p] = P.vind[q];
    P.vind[q] = t;
  }
};

// middleSplit_'s index from lim1 / lim2, and the two children (first child at
// next + 2 * split[j], split exclusively scanned)
struct KdChildrenFn {
  KdBuild B;
  int base;
  int next;
  const int* split;
  const int* scan0;
  const int* scan1;
  PCC_HD void operator()(int64_t j) const
  {
    const int64_t i = base + j;
    if (B.feat[i] < 0)
      return;
    const int32_t lo = B.lo[i], hi = B.hi[i];
    const int32_t count = hi - lo;
    const int32_t lim1 = scan0[hi] - scan0[lo];
    const int32_t lim2 = lim1 + scan1[hi] - scan1[lo + lim1];
    const int32_t index = lim1 > count / 2 ? lim1 : lim2 < count / 2 ? lim2 : count / 2;
    const int32_t c = next + 2 * split[j];
    const int f = B.feat[i];
    B.index[i] = index;
    B.child[i] = c;
    B.lo[c] = lo;
    B.hi[c] = lo + index;
    B.lo[c + 1] = lo + index;
    B.hi[c + 1] = hi;
    B.parent[c] = int32_t(i);
    B.parent[c + 1] = int32_t(i);
    for (int k = 0; k < 6; k++) {
      B.box[6 * size_t(c) + k] = B.box[6 * i + k];
      B.box[6 * size_t(c + 1) + k] = B.box[6 * i + k];
    }
    B.box[6 * size_t(c) + 3 + f] = B.cut[i];   // left: high = cutval
    B.box[6 * size_t(c + 1) + f] = B.cut[i];   // right: low = cutval
  }
};

// every point moves to its child on the next level, or leaves the build
struct KdSegFn {
  KdBuild B;
  int32_t* seg;
  PCC_HD void operator()(int64_t p) const
  {
    const int32_t s = seg[p];
    if (s < 0)
      return;
    if (B.feat[s] < 0)
      seg[p] = -1;
    else
      seg[p] = B.child[s] + (p - B.lo[s] >= B.index[s] ? 1 : 0);
  }
};

struct KdGatherFn {
  const int32_t* xyz;
  const int32_t* vind;
  int32_t* tpos;
  PCC_HD void operator()(int64_t i) const
  {
    for (int k = 0; k < 3; k++)
      tpos[3 * i + k] = xyz[3 * size_t(vind[i]) + k];
  }
};

// Builds nanoflann's tree over n points (xyz: executor memory, |x| < 2^30 --
// checked by the caller).  Returns a PCCB200_* status.
template<class Exec>
int
build_kdtree(Exec& ex, const int32_t* xyz, int n, KdTree& T)
{
  const int maxNodes = 2 * n;  // leaves <= n, so nodes <= 2n - 1
  KdBuild B;
  B.lo = ex.template alloc<int32_t>(maxNodes);
  B.hi = ex.template alloc<int32_t>(maxNodes);
  B.child = ex.template alloc<int32_t>(maxNodes);
  B.feat = ex.template alloc<int32_t>(maxNodes);
  B.parent = ex.template alloc<int32_t>(maxNodes);
  B.index = ex.template alloc<int32_t>(maxNodes);
  B.divLow = ex.template alloc<double>(maxNodes);
  B.divHigh = ex.template alloc<double>(maxNodes);
  B.cut = ex.template alloc<double>(maxNodes);
  B.box = ex.template alloc<double>(size_t(maxNodes) * 6);
  B.mn = ex.template alloc<int32_t>(size_t(maxNodes) * 3);
  B.mx = ex.template alloc<int32_t>(size_t(maxNodes) * 3);
  int32_t* vind = ex.template alloc<int32_t>(n);
  int32_t* seg = ex.template alloc<int32_t>(n);
  int* scan0 = ex.template alloc<int>(size_t(n) + 1);
  int* scan1 = ex.template alloc<int>(size_t(n) + 1);
  int32_t* slot = ex.template alloc<int32_t>(n);
  int* split = ex.template alloc<int>(size_t(n) + 1);  // a level has at most n nodes

  ex.foreach(n, KdInitFn{vind, seg});
  const int32_t root[3] = {0, n, -1};
  ex.upload(B.lo, &root[0], sizeof(int32_t));
  ex.upload(B.hi, &root[1], sizeof(int32_t));
  ex.upload(B.parent, &root[2], sizeof(int32_t));
  int begin = 0, end = 1, depth = 0;
  for (;;) {
    const int width = end - begin;
    ex.foreach(width, KdNodeInitFn{B, begin});
    ex.foreach(n, KdMinMaxFn{B, xyz, vind, seg});
    ex.foreach(width, KdSplitFn{B, begin, split});
    const KdPass p0{xyz, vind, seg, scan0, 0};
    ex.foreach(int64_t(n) + 1, KdFlagFn{B, p0, n, scan0});
    ex.exclusive_scan(scan0, int64_t(n) + 1);
    ex.foreach(n, KdPairRightFn{B, p0, scan0, slot});
    ex.foreach(n, KdPairLeftFn{B, p0, scan0, slot});
    const KdPass p1{xyz, vind, seg, scan0, 1};
    ex.foreach(int64_t(n) + 1, KdFlagFn{B, p1, n, scan1});
    ex.exclusive_scan(scan1, int64_t(n) + 1);
    ex.foreach(n, KdPairRightFn{B, p1, scan1, slot});
    ex.foreach(n, KdPairLeftFn{B, p1, scan1, slot});
    ex.zero(split + width, sizeof(int));
    ex.exclusive_scan(split, int64_t(width) + 1);
    ex.foreach(width, KdChildrenFn{B, begin, end, split, scan0, scan1});
    int splits = 0;
    ex.download(&splits, split + width, sizeof(int));
    if (splits == 0)
      break;
    ex.foreach(n, KdSegFn{B, seg});
    begin = end;
    end += 2 * splits;
    if (++depth > kKdMaxDepth)
      return PCCB200_ERR_UNSUPPORTED;
  }
  int32_t* tpos = ex.template alloc<int32_t>(size_t(n) * 3);
  ex.foreach(n, KdGatherFn{xyz, vind, tpos});
  int32_t rb[6];
  ex.download(rb, B.mn, 3 * sizeof(int32_t));
  ex.download(rb + 3, B.mx, 3 * sizeof(int32_t));
  T.vind = vind;
  T.tpos = tpos;
  T.child = B.child;
  T.lo = B.lo;
  T.hi = B.hi;
  T.feat = B.feat;
  T.divLow = B.divLow;
  T.divHigh = B.divHigh;
  for (int k = 0; k < 3; k++) {
    T.rootLow[k] = double(rb[k]);
    T.rootHigh[k] = double(rb[3 + k]);
  }
  T.n = n;
  T.numNodes = end;
  T.depth = depth;
  return PCCB200_OK;
}

//----------------------------------------------------------------------------
// the search: findNeighbors with a KNNResultSet and eps = 0

// nanoflann's KNNResultSet (without NANOFLANN_FIRST_MATCH): a new distance
// goes after the equal ones already held
struct KdResult {
  double d[kKdResultMax];
  int32_t id[kKdResultMax];
  int count;
  int cap;
  PCC_HD void init(int k)
  {
    cap = k;
    count = 0;
    d[k - 1] = DBL_MAX;
  }
  PCC_HD double worst() const { return d[cap - 1]; }
  PCC_HD void add(double dist, int32_t index)
  {
    int i;
    for (i = count; i > 0; --i) {
      if (d[i - 1] > dist) {
        if (i < cap) {
          d[i] = d[i - 1];
          id[i] = id[i - 1];
        }
      } else
        break;
    }
    if (i < cap) {
      d[i] = dist;
      id[i] = index;
    }
    if (count < cap)
      count++;
  }
};

// searchLevel with an explicit stack.  A frame is an internal node on the path
// whose best child is being searched (stage 0: node >= 0) or whose other child
// is (stage 1: ~node), with the node's mindistsq and the dists[divfeat] it has
// to restore.
PCC_HD void
kd_find_neighbours(const KdTree& T, const double q[3], KdResult& R)
{
  double dists[3] = {0.0, 0.0, 0.0};
  double mind = 0.0;  // computeInitialDistances
  for (int k = 0; k < 3; k++) {
    if (q[k] < T.rootLow[k]) {
      const double df = dsub(q[k], T.rootLow[k]);
      dists[k] = dmul(df, df);
      mind = dadd(mind, dists[k]);
    }
    if (q[k] > T.rootHigh[k]) {
      const double df = dsub(q[k], T.rootHigh[k]);
      dists[k] = dmul(df, df);
      mind = dadd(mind, dists[k]);
    }
  }
  int32_t stNode[kKdMaxDepth];
  double stMind[kKdMaxDepth];
  double stDst[kKdMaxDepth];
  int sp = 0;
  int32_t node = 0;
  for (;;) {
    // down the best children to a leaf
    for (int32_t c; (c = T.child[node]) >= 0;) {
      const int f = T.feat[node];
      const double diff1 = dsub(q[f], T.divLow[node]);
      const double diff2 = dsub(q[f], T.divHigh[node]);
      stNode[sp] = node;
      stMind[sp] = mind;
      stDst[sp] = dists[f];
      sp++;
      node = dadd(diff1, diff2) < 0 ? c : c + 1;
    }
    const double worst = R.worst();
    for (int32_t i = T.lo[node]; i < T.hi[node]; i++) {
      const int32_t* p = T.tpos + 3 * size_t(i);
      double dist = 0.0;
      for (int k = 0; k < 3; k++) {
        const double df = dsub(q[k], double(p[k]));
        dist = dadd(dist, dmul(df, df));
      }
      if (dist < worst)
        R.add(dist, T.vind[i]);
    }
    // back up to the next other child worth searching
    for (;;) {
      if (sp == 0)
        return;
      const int32_t top = stNode[sp - 1];
      const int32_t nd = top >= 0 ? top : ~top;
      const int f = T.feat[nd];
      if (top < 0) {  // the other child is done
        dists[f] = stDst[sp - 1];
        sp--;
        continue;
      }
      const double val = q[f];
      const double diff1 = dsub(val, T.divLow[nd]);
      const double diff2 = dsub(val, T.divHigh[nd]);
      const bool left = dadd(diff1, diff2) < 0;
      const double cb = dsub(val, left ? T.divHigh[nd] : T.divLow[nd]);
      const double cutDist = dmul(cb, cb);
      const double dst = stDst[sp - 1];
      const double m = dsub(dadd(stMind[sp - 1], cutDist), dst);
      dists[f] = cutDist;
      if (m <= R.worst()) {
        stNode[sp - 1] = ~nd;
        node = T.child[nd] + (left ? 1 : 0);
        mind = m;
        break;
      }
      dists[f] = dst;
      sp--;
    }
  }
}

//----------------------------------------------------------------------------
// libstdc++'s std::sort (introsort: median-of-three pivot moved to the front,
// unguarded partition, heap sort below depth 2 lg n, a final insertion sort
// with threshold 16), restated from the algorithm over the parallel arrays
// key / val, ordered by less(key a, key b) alone.  Equal keys end where this
// algorithm puts them, which is what the reference's backward lists depend on.

template<class K, class V, class Less>
struct GnuSort {
  K* key;
  V* val;
  Less less;

  PCC_HD void swap(int a, int b) const
  {
    const K k = key[a];
    key[a] = key[b];
    key[b] = k;
    const V v = val[a];
    val[a] = val[b];
    val[b] = v;
  }
  PCC_HD void move(int to, int from) const
  {
    key[to] = key[from];
    val[to] = val[from];
  }

  // __push_heap / __adjust_heap over [first, first + len)
  PCC_HD void adjust_heap(int first, int hole, int len, K vk, V vv) const
  {
    const int top = hole;
    int second = hole;
    while (second < (len - 1) / 2) {
      second = 2 * (second + 1);
      if (less(key[first + second], key[first + second - 1]))
        second--;
      move(first + hole, first + second);
      hole = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
      second = 2 * (second + 1);
      move(first + hole, first + second - 1);
      hole = second - 1;
    }
    int parent = (hole - 1) / 2;
    while (hole > top && less(key[first + parent], vk)) {
      move(first + hole, first + parent);
      hole = parent;
      parent = (hole - 1) / 2;
    }
    key[first + hole] = vk;
    val[first + hole] = vv;
  }

  // __partial_sort(first, last, last): make_heap, then sort_heap
  PCC_HD void heap_sort(int first, int last) const
  {
    const int len = last - first;
    if (len >= 2) {
      for (int parent = (len - 2) / 2;; parent--) {
        adjust_heap(first, parent, len, key[first + parent], val[first + parent]);
        if (parent == 0)
          break;
      }
    }
    while (last - first > 1) {
      --last;
      const K vk = key[last];
      const V vv = val[last];
      move(last, first);
      adjust_heap(first, 0, last - first, vk, vv);
    }
  }

  // __move_median_to_first(result, a, b, c)
  PCC_HD void median_to_first(int result, int a, int b, int c) const
  {
    if (less(key[a], key[b])) {
      if (less(key[b], key[c]))
        swap(result, b);
      else if (less(key[a], key[c]))
        swap(result, c);
      else
        swap(result, a);
    } else if (less(key[a], key[c]))
      swap(result, a);
    else if (less(key[b], key[c]))
      swap(result, c);
    else
      swap(result, b);
  }

  // __unguarded_partition_pivot
  PCC_HD int partition_pivot(int first, int last) const
  {
    const int mid = first + (last - first) / 2;
    median_to_first(first, first + 1, mid, last - 1);
    int lo = first + 1, hi = last;
    for (;;) {
      while (less(key[lo], key[first]))
        ++lo;
      --hi;
      while (less(key[first], key[hi]))
        --hi;
      if (!(lo < hi))
        return lo;
      swap(lo, hi);
      ++lo;
    }
  }

  // __unguarded_linear_insert
  PCC_HD void linear_insert(int last) const
  {
    const K vk = key[last];
    const V vv = val[last];
    int next = last - 1;
    while (less(vk, key[next])) {
      move(last, next);
      last = next;
      --next;
    }
    key[last] = vk;
    val[last] = vv;
  }

  // __insertion_sort
  PCC_HD void insertion_sort(int first, int last) const
  {
    if (first == last)
      return;
    for (int i = first + 1; i != last; ++i) {
      if (less(key[i], key[first])) {
        const K vk = key[i];
        const V vv = val[i];
        for (int j = i; j > first; j--)
          move(j, j - 1);
        key[first] = vk;
        val[first] = vv;
      } else
        linear_insert(i);
    }
  }

  PCC_HD void operator()(int n) const
  {
    if (n <= 1)
      return;
    // __introsort_loop; the recursion on the right part becomes a stack of
    // (first, last, depth), at most 2 lg n deep
    int stFirst[64], stLast[64], stDepth[64];
    int sp = 0;
    int lg = 0;
    while ((int64_t(2) << lg) <= n)
      lg++;
    stFirst[sp] = 0;
    stLast[sp] = n;
    stDepth[sp] = 2 * lg;
    sp++;
    while (sp > 0) {
      sp--;
      const int first = stFirst[sp];
      int last = stLast[sp];
      int depth = stDepth[sp];
      while (last - first > 16) {
        if (depth == 0) {
          heap_sort(first, last);
          break;
        }
        --depth;
        const int cut = partition_pivot(first, last);
        // __introsort_loop(cut, last) runs before the loop continues on
        // [first, cut); the two ranges are disjoint, so the order of the two
        // does not change the result
        stFirst[sp] = cut;
        stLast[sp] = last;
        stDepth[sp] = depth;
        sp++;
        last = cut;
      }
    }
    // __final_insertion_sort
    if (n > 16) {
      insertion_sort(0, 16);
      for (int i = 16; i != n; ++i)
        linear_insert(i);
    } else
      insertion_sort(0, n);
  }
};

struct DistLess {
  PCC_HD bool operator()(double a, double b) const { return a < b; }
};
struct IndexLess {
  PCC_HD bool operator()(int32_t a, int32_t b) const { return a < b; }
};

}  // namespace pccb200
