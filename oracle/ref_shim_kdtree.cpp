// ref_shim_kdtree.cpp — TEST INFRASTRUCTURE ONLY (oracle).
//
// extern "C" access to the UNMODIFIED nanoflann the reference recolours with
// (dependencies/nanoflann, through KDTreeVectorOfVectorsAdaptor<PCCPointSet3,
// double> with leaf size 10, as tmc3/pointset_processing.cpp builds it), and to
// the compiled std::sort the reference orders its backward lists with.  Built
// by `make -C oracle -f recolour_codec.mk kdtreeref` into
// oracle/_ref/libtmc13_kdtree.so.  Only tests/ may load it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "KDTreeVectorOfVectorsAdaptor.h"
#include "PCCPointSet.h"

using namespace pcc;

namespace {

typedef KDTreeVectorOfVectorsAdaptor<PCCPointSet3, double> Tree;
typedef Tree::index_t::Node Node;

PCCPointSet3
make_cloud(const int32_t* xyz, int n)
{
  PCCPointSet3 c;
  c.resize(n);
  for (int i = 0; i < n; i++)
    c[i] = point_t(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  return c;
}

// preorder: info[4 i..] = leaf?, lo, hi, divfeat (-1 for a leaf); div[2 i..] =
// divlow, divhigh (0 for a leaf).  An internal node's range is its subtree's.
int
preorder(const Node* node, int at, int32_t* info, double* div, int depth, int32_t* maxDepth)
{
  if (depth > *maxDepth)
    *maxDepth = depth;
  const bool leaf = !node->child1 && !node->child2;
  info[4 * at] = leaf;
  div[2 * at] = leaf ? 0.0 : node->node_type.sub.divlow;
  div[2 * at + 1] = leaf ? 0.0 : node->node_type.sub.divhigh;
  if (leaf) {
    info[4 * at + 1] = int32_t(node->node_type.lr.left);
    info[4 * at + 2] = int32_t(node->node_type.lr.right);
    info[4 * at + 3] = -1;
    return at + 1;
  }
  info[4 * at + 3] = node->node_type.sub.divfeat;
  const int c1 = at + 1;
  const int c2 = preorder(node->child1, c1, info, div, depth + 1, maxDepth);
  const int next = preorder(node->child2, c2, info, div, depth + 1, maxDepth);
  info[4 * at + 1] = info[4 * c1 + 1];
  info[4 * at + 2] = info[4 * c2 + 2];
  return next;
}

}  // namespace

// the tree over xyz (n x 3): vind (n), preorder nodes (at most 2n), root box;
// returns the node count
extern "C" int
ref_kdtree_build(const int32_t* xyz, int n, int32_t* vind, int32_t* info, double* div,
                 double* rootBox, int32_t* depth)
{
  const PCCPointSet3 cloud = make_cloud(xyz, n);
  Tree tree(3, cloud, 10);
  for (int i = 0; i < n; i++)
    vind[i] = int32_t(tree.index->vind[i]);
  for (int k = 0; k < 3; k++) {
    rootBox[k] = tree.index->root_bbox[k].low;
    rootBox[3 + k] = tree.index->root_bbox[k].high;
  }
  *depth = 0;
  return preorder(tree.index->root_node, 0, info, div, 0, depth);
}

// findNeighbors with a KNNResultSet<double> of k, as recolourColour queries
extern "C" int
ref_kdtree_knn(const int32_t* xyz, int n, const double* q, int nq, int k, int32_t* idx,
               double* dist)
{
  const PCCPointSet3 cloud = make_cloud(xyz, n);
  Tree tree(3, cloud, 10);
  nanoflann::KNNResultSet<double> rs(k);
  std::vector<size_t> ind(k);
  std::vector<double> d(k);
  for (int i = 0; i < nq; i++) {
    rs.init(&ind[0], &d[0]);
    tree.index->findNeighbors(rs, q + 3 * size_t(i), nanoflann::SearchParams(10));
    for (int j = 0; j < k; j++) {
      idx[size_t(i) * k + j] = j < int(rs.size()) ? int32_t(ind[j]) : -1;
      dist[size_t(i) * k + j] = j < int(rs.size()) ? d[j] : 0.0;
    }
  }
  return 0;
}

// std::sort of (key, val) pairs by key alone, as the backward lists are sorted
extern "C" void
ref_std_sort(double* key, int32_t* val, int n)
{
  struct Pair {
    double key;
    int32_t val;
  };
  std::vector<Pair> v(n);
  for (int i = 0; i < n; i++)
    v[i] = Pair{key[i], val[i]};
  std::sort(v.begin(), v.end(), [](const Pair& a, const Pair& b) { return a.key < b.key; });
  for (int i = 0; i < n; i++) {
    key[i] = v[i].key;
    val[i] = v[i].val;
  }
}
