// lod_pipeline.cuh — host-side schedule of one level-of-detail build, written
// against the executor concept of raht_pipeline.cuh (plus
// `morton_sort(xyz, n, keys, order)`), so that it drives CUDA kernels in the
// product and plain loops in the CPU unit tests.
//
// Mirrors buildPredictorsFast (tmc3/PCCTMC3Common.h:2300-2469) and
// AttributeLods::generate (tmc3/AttributeCommon.cpp:45-72): sort; per level
// subsample -> nearest neighbours of the refined points among the retained
// ones -> continue with the retained ones; finally updatePredictors,
// computeWeights, (blendWeights) and the coarse-to-fine index order.
#pragma once

#include <vector>

#include "lod_core.cuh"

namespace pccb200 {

// levels of detail of scalable lifting: one per octree level
// (AttributeParameterSet::maxNumDetailLevels, tmc3/hls.h:835-839)
constexpr int kScalableLevels = 21;

struct FillI32Fn {
  int* p;
  int v;
  PCC_HD void operator()(int64_t i) const { p[i] = v; }
};
struct CopyU32Fn {
  const uint32_t* src;
  uint32_t* dst;
  PCC_HD void operator()(int64_t i) const { dst[i] = src[i]; }
};

template<class Exec>
BoxHierarchy
build_boxes(Exec& ex, const int32_t* bpos, const uint32_t* list, int count)
{
  BoxHierarchy h;
  int c = count;
  const Box* lower = nullptr;
  for (int l = 0; l < 3; l++) {
    int below = c;
    c = (c + 31) >> 5;
    Box* b = ex.template alloc<Box>(c > 0 ? c : 1);
    ex.foreach(c, BoxLevelFn{bpos, l == 0 ? list : nullptr, lower, below, b});
    h.lvl[l] = b;
    lower = b;
  }
  return h;
}

// xyz: N x 3 in executor memory.  predsOut / indexesOut: executor memory.
// nplOut (host, PCCB200_MAX_LODS entries) / lodCountOut (host).
// scal: scalable lifting (scalable_lifting_enabled_flag), or null.  Then
// lp.num_detail_levels and lp.dist2 are not read: the levels are the octree
// levels min_geom_node_size_log2 .. 20 (maxNumDetailLevels(), tmc3/hls.h:835-839).
template<class Exec>
int
lod_run(Exec& ex, const pccb200_lod_params& lp, const int32_t* xyz, int N,
        pccb200_predictor* predsOut, uint32_t* indexesOut, uint32_t* nplOut, int* lodCountOut,
        const pccb200_lod_scalable* scal = nullptr)
{
  if (N <= 0 || lp.num_pred_nearest_neighbours < 1 || lp.num_pred_nearest_neighbours > 3
      || lp.lod_decimation_type < 0 || lp.lod_decimation_type > 2)
    return PCCB200_ERR_INVALID_ARG;
  if (scal) {
    if (lp.lod_decimation_type != 0 || scal->max_neigh_range < 1
        || scal->min_geom_node_size_log2 < 0 || scal->min_geom_node_size_log2 >= kScalableLevels
        || (scal->geom_num_points != 0 && scal->geom_num_points < N))
      return PCCB200_ERR_INVALID_ARG;
  } else {
    if (lp.num_detail_levels < 1 || lp.num_detail_levels > PCCB200_MAX_LODS)
      return PCCB200_ERR_INVALID_ARG;
    // cell shifts are 3 * (dist2 + lod + 1) bits of a 63-bit Morton code
    if (lp.lod_decimation_type != 1
        && (lp.dist2 < 0 || lp.dist2 + lp.num_detail_levels > 20))
      return PCCB200_ERR_INVALID_ARG;
    if (lp.lod_decimation_type != 0)
      for (int l = 0; l + 1 < lp.num_detail_levels; l++)
        if (lp.lod_sampling_period[l] < 2)
          return PCCB200_ERR_INVALID_ARG;
  }
  LodConfig cfg;
  cfg.numDetailLevels = scal ? kScalableLevels : lp.num_detail_levels;
  cfg.decimation = lp.lod_decimation_type;
  for (int i = 0; i < PCCB200_MAX_LODS; i++)
    cfg.samplingPeriod[i] = lp.lod_sampling_period[i];
  cfg.dist2 = scal ? 0 : lp.dist2;
  cfg.numNeighbours = lp.num_pred_nearest_neighbours;
  cfg.interRange = lp.inter_lod_search_range;
  cfg.intraRange = lp.intra_lod_search_range;
  cfg.intraSkipLayers = lp.intra_lod_prediction_skip_layers;
  cfg.distribution = lp.prediction_with_distribution != 0;
  for (int k = 0; k < 3; k++)
    cfg.bias[k] = lp.lod_neigh_bias[k];
  cfg.blending = lp.pred_weight_blending != 0;
  cfg.maxNeighRange = scal ? scal->max_neigh_range : 0;

  ex.phase(0);
  int64_t* code = ex.template alloc<int64_t>(N);
  int32_t* order = ex.template alloc<int32_t>(N);
  ex.morton_sort(xyz, N, code, order);
  ex.phase(5);
  int32_t* pos = ex.template alloc<int32_t>(size_t(N) * 3);
  int32_t* bpos = ex.template alloc<int32_t>(size_t(N) * 3);
  VoxelGatherFn vg;
  vg.xyz = xyz;
  vg.order = order;
  for (int k = 0; k < 3; k++)
    vg.bias[k] = cfg.bias[k];
  vg.pos = pos;
  vg.bpos = bpos;
  ex.foreach(N, vg);
  Voxels v{N, code, pos, bpos, order};

  uint32_t* input = ex.template alloc<uint32_t>(N);
  uint32_t* retained = ex.template alloc<uint32_t>(N);
  // refined entries of every level in build order (buildPredictorsFast's
  // indexes before they become point indices): the concatenation of scalable
  // lifting searches the earlier levels again
  uint32_t* refined = ex.template alloc<uint32_t>(N);
  uint32_t* indexesBuild = ex.template alloc<uint32_t>(N);
  uint8_t* keep = ex.template alloc<uint8_t>(N);
  int32_t* cellFirst = ex.template alloc<int32_t>(size_t(N) + 1);
  int32_t* segFirst = ex.template alloc<int32_t>(size_t(N) + 1);
  int* decision = ex.template alloc<int>(N);
  // centroid mode: jump tables of the segmentation, one per doubling level
  int jumpLevels = 1;
  while ((int64_t(1) << jumpLevels) < N)
    jumpLevels++;
  int32_t* jump =
    cfg.decimation == 2 ? ex.template alloc<int32_t>(size_t(N) * jumpLevels) : nullptr;
  int* dCount = ex.template alloc<int>(4);
  unsigned long long* dStuck = ex.template alloc<unsigned long long>(1);
  uint32_t* p2p = ex.template alloc<uint32_t>(N);
  uint32_t* predCount = ex.template alloc<uint32_t>(N);
  uint32_t* predIdx = ex.template alloc<uint32_t>(size_t(N) * 3);
  uint64_t* predW = ex.template alloc<uint64_t>(size_t(N) * 3);
  ex.foreach(N, IotaFn{input});

  std::vector<uint32_t> npl;
  npl.push_back(uint32_t(N));
  int nInput = N, nIndexes = 0, predBase = N;

  // nearest neighbours of the refined entries queries[0, nQ) of level `lod`
  // among the retained ones; their predictor slots are predBase - 1 down
  auto search = [&](int lod, const uint32_t* queries, int nQ, int start, const uint32_t* ret,
                    int nRet) {
    ex.phase(2);  // (profiling tag: neighbour search)
    if (scal)
      ex.foreach(N, BiasMaskFn{pos, {cfg.bias[0], cfg.bias[1], cfg.bias[2]}, lod, bpos});
    KnnFn kn;
    kn.cfg = cfg;
    kn.v = v;
    kn.retained = ret;
    kn.R = nRet;
    kn.queries = queries;
    kn.nQueries = nQ;
    kn.lod = lod;
    kn.hb = build_boxes(ex, bpos, ret, nRet);
    if (lod >= cfg.intraSkipLayers)
      kn.hq = build_boxes(ex, bpos, queries, nQ);
    else
      kn.hq = kn.hb;
    unsigned long long none = ~0ull;
    ex.upload(dStuck, &none, sizeof(none));
    const int sb3 = 3 * (1 + cfg.dist2 + lod);
    ex.foreach(nRet, StuckAtlasFn{code, ret, queries, nQ, sb3 + 21 < 63 ? sb3 + 21 : 63, dStuck});
    kn.stuck = dStuck;
    kn.predBase = predBase;
    kn.indexesOut = indexesBuild + start;
    kn.p2p = p2p;
    kn.predCount = predCount;
    kn.predIdx = predIdx;
    kn.predW = predW;
    ex.foreach(nQ, kn);
    predBase -= nQ;
  };

  const int L = cfg.numDetailLevels;
  const int lod0 = scal ? scal->min_geom_node_size_log2 : 0;
  // scalable lifting: layers are concatenated while a level refines more
  // points than the earlier levels and the skipped points together
  // (PCCTMC3Common.h:2377-2406)
  bool concatenate = scal != nullptr;
  const int64_t skipped = scal && scal->geom_num_points ? scal->geom_num_points - N : 0;
  for (int lod = lod0; nInput > 0 && lod < L; lod++) {
    const int start = nIndexes;
    uint32_t* queries = refined + start;
    int nRet = 0, nQ = 0;
    ex.phase(1);  // (profiling tag: subsampling)
    if (lod == L - 1 || nInput == 1 && cfg.decimation != 1) {
      // last level, or a single point left: everything is refined
      ex.foreach(nInput, CopyU32Fn{input, queries});
      nQ = nInput;
    } else if (cfg.decimation == 1) {
      const int period = cfg.samplingPeriod[lod];
      nRet = period > 0 ? (nInput + period - 1) / period : 0;
      nQ = nInput - nRet;
      ex.foreach(nInput, SubsamplePeriodicFn{input, retained, queries, period});
    } else {
      // cells / octree nodes: runs of equal (code >> shift)
      const int shift = 3 * (cfg.dist2 + lod + 1);
      ex.compact(nInput, CellHead{code, input, shift}, CellEmit{cellFirst}, dCount);
      int nCells = 0;
      ex.download(&nCells, dCount, sizeof(int));
      int32_t n32 = nInput;
      ex.upload(cellFirst + nCells, &n32, sizeof(int32_t));
      if (scal) {
        // subsampleByOctree, period 0: every octree node is a segment
        ex.foreach(nCells, CentroidPickFn{v, input, cellFirst, lod, (lod & 1) != 0, keep});
      } else if (cfg.decimation == 0) {
        ex.foreach(nCells, FillI32Fn{decision, kCellUndecided});
        SubsampleDistanceFn fn;
        fn.v = v;
        fn.input = input;
        fn.nInput = nInput;
        fn.cellFirst = cellFirst;
        fn.nCells = nCells;
        fn.shiftBits0 = cfg.dist2 + lod;
        fn.decision = decision;
        fn.keep = keep;
        ex.subsample_distance(fn, nCells);
      } else {
        // segment starts = groups reachable from group 0 (see CentroidNextFn)
        int levels = 1;
        while ((int64_t(1) << levels) < nCells)
          levels++;
        ex.foreach(nCells, CentroidNextFn{cellFirst, nCells, cfg.samplingPeriod[lod], jump});
        for (int i = 1; i < levels; i++)
          ex.foreach(nCells, JumpSquareFn{jump + size_t(i - 1) * N, jump + size_t(i) * N, nCells});
        uint8_t* mark = reinterpret_cast<uint8_t*>(decision);
        ex.zero(mark, size_t(nCells));
        const uint8_t one = 1;
        ex.upload(mark, &one, 1);
        for (int i = levels - 1; i >= 0; i--)
          ex.foreach(nCells, JumpMarkFn{jump + size_t(i) * N, mark, nCells});
        ex.compact(nCells, MarkPred{mark}, SegmentEmit{cellFirst, segFirst}, dCount + 1);
        int nSeg = 0;
        ex.download(&nSeg, dCount + 1, sizeof(int));
        ex.upload(segFirst + nSeg, &n32, sizeof(int32_t));
        ex.foreach(nSeg, CentroidPickFn{v, input, segFirst, cfg.dist2 + lod, true, keep});
      }
      ex.compact(nInput, KeepPred{keep, 1}, ListEmit{input, retained}, dCount + 2);
      ex.compact(nInput, KeepPred{keep, 0}, ListEmit{input, queries}, dCount + 3);
      int counts[2];
      ex.download(counts, dCount + 2, 2 * sizeof(int));
      nRet = counts[0];
      nQ = counts[1];
    }
    nIndexes += nQ;

    if (concatenate && nQ > 0) {
      if (nQ <= start + skipped) {
        concatenate = false;
      } else {
        // the earlier levels, each at its own lodIndex, against this level's
        // retained points; their predictor slots are assigned again
        predBase = N;
        for (int e = 0; e + 1 < int(npl.size()); e++) {
          const int s0 = N - int(npl[e]), s1 = N - int(npl[e + 1]);
          if (s1 > s0)
            search(lod0 + e, refined + s0, s1 - s0, s0, retained, nRet);
        }
      }
    }
    // nearest neighbours of the refined points among the retained ones
    if (nQ > 0)
      search(lod, queries, nQ, start, retained, nRet);
    if (nRet)
      npl.push_back(uint32_t(nRet));
    uint32_t* t = input;
    input = retained;
    retained = t;
    nInput = nRet;
  }

  ex.phase(3);  // (profiling tag: finalisation)
  FinalizePredictorFn fin;
  fin.n = N;
  fin.blending = cfg.blending;
  fin.predCount = predCount;
  fin.predIdx = predIdx;
  fin.predW = predW;
  fin.p2p = p2p;
  fin.indexesBuild = indexesBuild;
  fin.xyz = xyz;
  fin.out = predsOut;
  fin.indexesOut = indexesOut;
  ex.foreach(N, fin);

  *lodCountOut = int(npl.size());
  for (size_t i = 0; i < npl.size(); i++)
    nplOut[i] = npl[npl.size() - 1 - i];
  return PCCB200_OK;
}

}  // namespace pccb200
