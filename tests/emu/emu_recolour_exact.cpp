// emu_recolour_exact.cpp — TEST INFRASTRUCTURE ONLY: the reference-exact
// recolouring bodies of the product (kdtree.cuh, recolour.cuh with
// kRecolourRefExact) compiled for the host and run as loops (see exec_host.h).
// Built by tests/test_recolour_exact.py into a temporary directory.
#include <vector>

#include "exec_host.h"
#include "recolour.cuh"

using namespace pccb200;

namespace {

// the tree in preorder, as oracle/ref_shim_kdtree.cpp writes nanoflann's:
// info[4 i..]: leaf?, lo, hi, divfeat (-1 for a leaf); div[2 i..]: divlow,
// divhigh (0 for a leaf)
int
preorder(const KdTree& T, const std::vector<int32_t>& child, const std::vector<int32_t>& lo,
         const std::vector<int32_t>& hi, const std::vector<int32_t>& feat,
         const std::vector<double>& dl, const std::vector<double>& dh, int node, int at,
         int32_t* info, double* div)
{
  const bool leaf = child[node] < 0;
  info[4 * at] = leaf;
  info[4 * at + 1] = lo[node];
  info[4 * at + 2] = hi[node];
  info[4 * at + 3] = leaf ? -1 : feat[node];
  div[2 * at] = leaf ? 0.0 : dl[node];
  div[2 * at + 1] = leaf ? 0.0 : dh[node];
  int next = at + 1;
  if (!leaf) {
    next = preorder(T, child, lo, hi, feat, dl, dh, child[node], next, info, div);
    next = preorder(T, child, lo, hi, feat, dl, dh, child[node] + 1, next, info, div);
  }
  return next;
}

}  // namespace

// nanoflann's tree over xyz (n x 3): vind (n), the preorder node list (at most
// 2n nodes); returns the node count, or -1
extern "C" int
emu_kdtree_build(const int32_t* xyz, int n, int32_t* vind, int32_t* info, double* div,
                 double* rootBox, int32_t* depth)
{
  HostExec ex;
  KdTree T;
  if (build_kdtree(ex, xyz, n, T) != PCCB200_OK)
    return -1;
  std::vector<int32_t> child(T.child, T.child + T.numNodes), lo(T.lo, T.lo + T.numNodes),
    hi(T.hi, T.hi + T.numNodes), feat(T.feat, T.feat + T.numNodes);
  std::vector<double> dl(T.divLow, T.divLow + T.numNodes), dh(T.divHigh, T.divHigh + T.numNodes);
  for (int i = 0; i < n; i++)
    vind[i] = T.vind[i];
  for (int k = 0; k < 3; k++) {
    rootBox[k] = T.rootLow[k];
    rootBox[3 + k] = T.rootHigh[k];
  }
  *depth = T.depth;
  return preorder(T, child, lo, hi, feat, dl, dh, 0, 0, info, div);
}

// findNeighbors on the tree over xyz for nq query points q (nq x 3, double)
extern "C" int
emu_kdtree_knn(const int32_t* xyz, int n, const double* q, int nq, int k, int32_t* idx,
               double* dist)
{
  HostExec ex;
  KdTree T;
  if (k < 1 || k > kKdResultMax || build_kdtree(ex, xyz, n, T) != PCCB200_OK)
    return -1;
  for (int i = 0; i < nq; i++) {
    KdResult R;
    R.init(k);
    kd_find_neighbours(T, q + 3 * size_t(i), R);
    for (int j = 0; j < k; j++) {
      idx[size_t(i) * k + j] = j < R.count ? R.id[j] : -1;
      dist[size_t(i) * k + j] = j < R.count ? R.d[j] : 0.0;
    }
  }
  return 0;
}

// the std::sort restatement: (key, val) pairs ordered by key alone
extern "C" void
emu_gnu_sort(double* key, int32_t* val, int n)
{
  GnuSort<double, int32_t, DistLess>{key, val, DistLess{}}(n);
}

extern "C" int
emu_recolour_exact(const pccb200_recolour_params* rp, const int32_t* srcXyz,
                   const int32_t* srcAttr, int A, int nSrc, double scale, const int32_t* off,
                   const int32_t* tgtXyz, int nTgt, int bitdepth, int32_t* out)
{
  HostExec ex;
  return recolour_run(ex, *rp, srcXyz, srcAttr, A, nSrc, scale, off, tgtXyz, nTgt, bitdepth, out,
                      kRecolourRefExact);
}

// the grid path on the same inputs (the lowest-index rule the exact path
// departs from)
extern "C" int
emu_recolour_grid(const pccb200_recolour_params* rp, const int32_t* srcXyz,
                  const int32_t* srcAttr, int A, int nSrc, double scale, const int32_t* off,
                  const int32_t* tgtXyz, int nTgt, int bitdepth, int32_t* out)
{
  HostExec ex;
  return recolour_run(ex, *rp, srcXyz, srcAttr, A, nSrc, scale, off, tgtXyz, nTgt, bitdepth, out);
}
