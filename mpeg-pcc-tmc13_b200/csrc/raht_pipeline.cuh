// raht_pipeline.cuh — the host-side schedule of one RAHT call, written
// against an executor so that the same schedule drives CUDA kernels
// (exec_cuda.cuh: DeviceExec) and, for the CPU unit tests of the kernel
// bodies, plain loops (tests/emu/exec_host.h: HostExec).
//
// Executor concept:
//   T*   alloc<T>(size_t n)                 workspace memory (uninitialised)
//   void phase(int p)                        tag following launches (profiling)
//   void zero(void* p, size_t bytes);  void fill(void* p, int byte, size_t bytes)
//   void upload(void* dst, const void* src, size_t bytes)      host -> exec
//   void download(void* dst, const void* src, size_t bytes)    exec -> host, synchronous
//   void foreach(int64_t n, F f)            f(i) for i in [0, n), any order
//   void ordered(int64_t n, F f)            f(i) with block-level dataflow:
//                                           f may spin on flags set by f(j), j < i
//   void compact(int64_t n, Pred p, Emit e, int* total = nullptr)
//                                           e(rank, i) for every i with p(i),
//                                           rank = number of j < i with p(j);
//                                           *total (executor memory) = count
//   void subsample_distance(SubsampleDistanceFn fn, int nCells)   (lod_pipeline.cuh)
//   void block_stage(BlockFn fn, int64_t nBlocks, int* tzNext)
//                                           one top-down stage with the
//                                           thread-per-block body, then the
//                                           zero-run counter to tzNext;
//                                           the stages of a descent WaveDescent
//                                           (below) does not take
//
// Mirrors the control flow of uraht_process (tmc3/RAHT.cpp:977-1976).
#pragma once

#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "raht_core.cuh"

namespace pccb200 {

// An executor may provide its own schedule of the whole descent (specialised
// for the CUDA executor in raht_wave.cuh); the generic one below walks the
// stages through Exec::block_stage.
template<class Exec>
struct WaveDescent {
  static constexpr bool available = false;
  struct Job {};
};

struct StagePlan {
  int level;
  int n;
};

// Stage levels from the adjacent-key histogram: every third binary level
// below the first level at which all points agree; a level that adds no
// nodes with respect to the level above is skipped (RAHT.cpp:1086,1205-1209).
// Returns the stages fine -> coarse; empty when all points coincide.
inline std::vector<StagePlan>
plan_stages(const int hist[64], int& nLeaves)
{
  int64_t total = 0;
  int top = -1;
  for (int h = 0; h < 64; h++) {
    total += hist[h];
    if (hist[h])
      top = h;
  }
  nLeaves = int(total + 1);
  std::vector<StagePlan> stages;
  if (top < 0)
    return stages;
  const int lmax = top + 1;
  const int rootLevel = 3 * ((lmax - 1) / 3);
  auto count = [&](int s) {
    int64_t c = 1;
    for (int h = s; h < 64; h++)
      c += hist[h];
    return int(c);
  };
  for (int s = 0; s <= rootLevel; s += 3) {
    int c = count(s);
    if (s == rootLevel || c != count(s + 3)) {
      if (stages.empty())
        c = nLeaves;  // the finest processed stage holds the leaves
      stages.push_back({s, c});
    }
  }
  return stages;
}

template<class Exec>
Stage
alloc_stage(Exec& ex, int level, int n, int A, bool hasQp, bool needRec)
{
  Stage s;
  s.level = level;
  s.n = n;
  s.key = ex.template alloc<int64_t>(n);
  s.weight = ex.template alloc<int32_t>(n);
  s.attr = ex.template alloc<int32_t>(size_t(n) * A);
  s.qpUp = hasQp ? ex.template alloc<int32_t>(size_t(n) * 2) : nullptr;
  s.qpDown = hasQp ? ex.template alloc<int32_t>(size_t(n) * 2) : nullptr;
  s.first = ex.template alloc<int32_t>(size_t(n) + 1);
  s.nn = ex.template alloc<int32_t>(n);
  s.occ = ex.template alloc<uint8_t>(n);
  s.rec = needRec ? ex.template alloc<int64_t>(size_t(n) * A) : nullptr;
  s.recUs = needRec ? ex.template alloc<int64_t>(size_t(n) * A) : nullptr;
  s.done = ex.template alloc<int>(n);
  return s;
}

inline RahtConfig
make_config(const pccb200_raht_params& pp, const pccb200_qpset& qs, bool forward,
            int A, bool hasQp)
{
  RahtConfig c;
  c.A = A;
  c.isEncoder = forward;
  c.ext = pp.raht_extension != 0;
  c.haar = pp.integer_haar != 0;
  c.hasQp = hasQp;
  c.predictionEnabled = pp.prediction_enabled != 0;
  c.subnode = pp.subnode_prediction_enabled != 0;
  c.thr0 = pp.prediction_threshold0;
  c.thr1 = pp.prediction_threshold1;
  c.searchRange = pp.prediction_search_range;
  for (int i = 0; i < 19; i++)
    c.predWeightParent[i] = pp.pred_weight_parent[i];
  for (int i = 0; i < 12; i++)
    c.predWeightChild[i] = pp.pred_weight_child[i];
  c.numLayers = qs.num_layers;
  c.maxQp = qs.max_qp;
  c.fixedPointQpOffset = qs.fixed_point_qp_offset;
  c.numAcLayers = qs.num_ac_coeff_qp_layers;
  return c;
}

// One attribute of a call: its quantisation parameters and coefficient planes
// (executor memory; component kk at coef + kk * coefStride).
struct RahtSetIO {
  const pccb200_qpset* qs;
  int A;
  int32_t* coef;
  int64_t coefStride;
};

// what a set needs at run time, for the executor's descent and the tail
struct RahtSetRt {
  int A, base;
  int numLayers, maxQp, fixedPointQpOffset, numAcLayers;
  const QpTables* qt;
  int32_t* coef;
  int64_t coefStride;
};

// A call whose descent and tail have been prepared but not run yet: the
// caller issues the descents of several such units together (one launch per
// descent step for all of them, WaveDescent<Exec>::run_gang) and then
// ex.foreach(nLeaves, tail) for each.  Only executors with their own descent
// can defer.
template<class Exec>
struct RahtDeferred {
  bool pending = false;
  typename WaveDescent<Exec>::Job job;
  TailFn tail;
  int nLeaves = 0;
};

// keys / attrs / qpo / coefficients live in executor memory.  attrs: N rows of
// all components of all sets (set 0 first), in and out.  Several sets = several
// attributes coded on the same positions in one pass: they share the tree and
// every geometry-only step; that needs the executor's own descent
// (WaveDescent) and returns PCCB200_ERR_UNSUPPORTED where it cannot be used
// (the caller codes such attributes one by one).  With defer, a descent
// WaveDescent runs is left prepared in *defer (pending) together with the
// tail; everything else runs here.  Returns a PCCB200_* status.
template<class Exec>
int
raht_run_sets(Exec& ex, const pccb200_raht_params& pp, int numSets, const RahtSetIO* io,
              bool forward, const int64_t* keys, int32_t* attrs, const int32_t* qpo, int N,
              RahtDeferred<Exec>* defer = nullptr)
{
  if (defer)
    defer->pending = false;
  if (N <= 0 || numSets < 1 || numSets > 2)
    return PCCB200_ERR_INVALID_ARG;
  int A = 0;
  for (int s = 0; s < numSets; s++) {
    const pccb200_qpset& qs = *io[s].qs;
    if (io[s].A < 1 || io[s].A > 3 || qs.num_layers < 1 || qs.num_layers > PCCB200_MAX_QP_LAYERS
        || qs.num_ac_coeff_qp_layers > PCCB200_MAX_AC_QP_LAYERS || qs.num_ac_coeff_qp_layers < 0)
      return PCCB200_ERR_INVALID_ARG;
    A += io[s].A;
  }
  if (A > 4)
    return PCCB200_ERR_INVALID_ARG;

  const bool hasQp = qpo != nullptr;
  const pccb200_qpset& qs = *io[0].qs;
  RahtConfig cfg = make_config(pp, qs, forward, A, hasQp);
  if (numSets > 1) {
    bool ok = N >= 2 && !hasQp;
    if constexpr (WaveDescent<Exec>::available) {
      for (int s = 0; s < numSets && ok; s++) {
        RahtConfig c1 = make_config(pp, *io[s].qs, forward, io[s].A, hasQp);
        ok = WaveDescent<Exec>::enabled(c1);
      }
    } else {
      ok = false;
    }
    if (!ok)
      return PCCB200_ERR_UNSUPPORTED;
  }

  RahtSetRt rt[2] = {};
  for (int s = 0, base = 0; s < numSets; base += io[s].A, s++) {
    const pccb200_qpset& q = *io[s].qs;
    QpTables hostQt;
    for (int i = 0; i < PCCB200_MAX_QP_LAYERS; i++) {
      hostQt.layers[i][0] = q.layers[i][0];
      hostQt.layers[i][1] = q.layers[i][1];
    }
    for (int l = 0; l < PCCB200_MAX_AC_QP_LAYERS; l++)
      for (int c = 0; c < 7; c++) {
        hostQt.acQps[l][c][0] = q.ac_coeff_qps[l][c][0];
        hostQt.acQps[l][c][1] = q.ac_coeff_qps[l][c][1];
      }
    QpTables* dq = ex.template alloc<QpTables>(1);
    ex.upload(dq, &hostQt, sizeof(QpTables));
    rt[s].A = io[s].A;
    rt[s].base = base;
    rt[s].numLayers = q.num_layers;
    rt[s].maxQp = q.max_qp;
    rt[s].fixedPointQpOffset = q.fixed_point_qp_offset;
    rt[s].numAcLayers = q.num_ac_coeff_qp_layers;
    rt[s].qt = dq;
    rt[s].coef = io[s].coef;
    rt[s].coefStride = io[s].coefStride;
  }
  const QpTables* qt = rt[0].qt;
  int32_t* coef = io[0].coef;
  const int64_t coefStride = io[0].coefStride;

  ex.phase(1);  // tree build
  if (N == 1) {
    ex.foreach(1, SinglePointFn{cfg, qt, qpo, attrs, coef, coefStride});
    return PCCB200_OK;
  }

  //-- adjacent-key statistics (one small synchronising read-back per call)
  int* dHist = ex.template alloc<int>(65);
  ex.zero(dHist, 65 * sizeof(int));
  ex.foreach(N, LevelHistFn{keys, dHist});
  int hist[65];
  ex.download(hist, dHist, sizeof(hist));
  if (hist[64])
    return PCCB200_ERR_UNSORTED;

  int nLeaves = 0;
  std::vector<StagePlan> plan = plan_stages(hist, nLeaves);
  const bool hasStages = !plan.empty();
  const int numDup = N - nLeaves;
  if (getenv("PCCB200_DEBUG")) {
    fprintf(stderr, "[pccb200] N=%d leaves=%d stages:", N, nLeaves);
    for (auto& st : plan)
      fprintf(stderr, " L%d:%d", st.level, st.n);
    fprintf(stderr, "\n");
  }

  //-- leaves
  std::vector<Stage> stages;
  Stage L = alloc_stage(ex, hasStages ? plan[0].level : 0, nLeaves, A, hasQp, true);
  stages.push_back(L);
  ex.compact(N, LeafHead{keys}, StageEmit{keys, L.key, L.first});
  {
    int32_t n32 = N;
    ex.upload(L.first + nLeaves, &n32, sizeof(int32_t));
  }
  int32_t* dupHf = nullptr;
  if (cfg.haar && numDup)
    dupHf = ex.template alloc<int32_t>(size_t(N) * A);
  ex.foreach(nLeaves, LeafFn{L, attrs, qpo, dupHf, A, cfg.haar});

  //-- coarser stages, bottom-up
  for (size_t i = 1; i < plan.size(); i++) {
    Stage& F = stages.back();
    Stage C = alloc_stage(ex, plan[i].level, plan[i].n, A, hasQp, true);
    ex.compact(F.n, StageHead{F.key, F.level + 3}, StageEmit{F.key, C.key, C.first});
    int32_t n32 = F.n;
    ex.upload(C.first + C.n, &n32, sizeof(int32_t));
    ex.foreach(C.n, MergeFn{F, C, A, cfg.haar});
    stages.push_back(C);
  }

  //-- descent, coarse to fine
  ex.phase(2);  // block transform
  int qpLayer = 0;
  bool descended = false;
  if constexpr (WaveDescent<Exec>::available) {
    if (hasStages && (numSets > 1 || WaveDescent<Exec>::enabled(cfg))) {
      typename WaveDescent<Exec>::Job local;
      typename WaveDescent<Exec>::Job* job = defer ? &defer->job : &local;
      WaveDescent<Exec>::prepare(ex, cfg, numSets, rt, stages, *job);
      if (defer)
        defer->pending = true;
      else
        WaveDescent<Exec>::run_gang(ex, &job, 1);
      descended = true;
    }
  }
  if (hasStages && !descended) {
    // one set (several need WaveDescent).  Zero-run look-back words: a region
    // of (blocks + 1) words per stage; word 0 of a region is the counter
    // handed over by the previous stage
    const bool rdoq = forward && !cfg.haar;
    std::vector<int64_t> tzOff(stages.size() + 1, 0);
    int* tz = nullptr;
    if (rdoq) {
      int64_t total = 0;
      for (int si = int(stages.size()) - 1; si >= 0; si--) {
        tzOff[si] = total;
        total += (si == int(stages.size()) - 1 ? 1 : stages[si + 1].n) + 1;
      }
      total++;
      tz = ex.template alloc<int>(size_t(total));
      ex.zero(tz, size_t(total) * sizeof(int));
      int init = tz_pack(kTzExit, 0);
      ex.upload(tz + tzOff[stages.size() - 1], &init, sizeof(int));
    }

    int acLayer = -1;
    for (int si = int(stages.size()) - 1; si >= 0; si--) {
      qpLayer = qpLayer + 1 < qs.num_layers ? qpLayer + 1 : qs.num_layers - 1;
      acLayer++;
      BlockFn fn;
      fn.cfg = cfg;
      fn.qt = qt;
      fn.S = stages[si];
      fn.coef = coef;
      fn.coefStride = coefStride;
      fn.qpLayer = qpLayer;
      fn.acLayer = acLayer;
      fn.tz = tz ? tz + tzOff[si] : nullptr;
      fn.useFlags = 1;
      const bool isRoot = si == int(stages.size()) - 1;
      if (isRoot) {
        fn.P = Stage{};
        fn.P.n = 0;
        fn.coefBase = 0;
        fn.predInLvl = 0;
      } else {
        fn.P = stages[si + 1];
        fn.coefBase = fn.P.n;
        fn.predInLvl = cfg.predictionEnabled;
        ex.zero(fn.P.done, size_t(fn.P.n) * sizeof(int));
      }
      // every reconstruction slot of the stage starts as "not ready"
      ex.fill(fn.S.rec, 0x80, size_t(fn.S.n) * A * sizeof(int64_t));
      // the executor runs the stage (single-child fast path + ordered
      // dataflow over the transforming blocks) and hands the zero-run
      // counter to the next stage's region
      int* tzNext = (tz && si > 0) ? tz + tzOff[si - 1] : nullptr;
      ex.block_stage(fn, isRoot ? 1 : fn.P.n, tzNext);
    }
  }

  //-- duplicates + write-back
  ex.phase(3);
  TailFn tail;
  tail.cfg = cfg;
  tail.numSets = numSets;
  for (int s = 0; s < numSets; s++) {
    TailSet& ts = tail.set[s];
    ts.A = rt[s].A;
    ts.base = rt[s].base;
    ts.maxQp = rt[s].maxQp;
    ts.fixedPointQpOffset = rt[s].fixedPointQpOffset;
    // the qp layer of the last stage: one step per stage, saturating
    const int steps = hasStages ? int(stages.size()) : 0;
    ts.qpLayer = steps < rt[s].numLayers - 1 ? steps : rt[s].numLayers - 1;
    if (ts.qpLayer < 0)
      ts.qpLayer = 0;
    ts.qt = rt[s].qt;
    ts.coef = rt[s].coef;
    ts.coefStride = rt[s].coefStride;
  }
  tail.L = stages[0];
  tail.attrsIn = attrs;
  tail.dupHf = dupHf;
  tail.attrsOut = attrs;
  tail.coefBase = hasStages ? nLeaves : 0;
  tail.hasStages = hasStages;
  if (defer && defer->pending) {
    defer->tail = tail;
    defer->nLeaves = nLeaves;
    return PCCB200_OK;
  }
  ex.foreach(nLeaves, tail);
  if (forward && !hasStages) {
    // all points coincide: the reference codes N-1 coefficients and no DC;
    // the last slot of each component is defined as zero here
    int32_t z = 0;
    for (int s = 0; s < numSets; s++)
      for (int k = 0; k < rt[s].A; k++)
        ex.upload(rt[s].coef + k * rt[s].coefStride + (N - 1), &z, sizeof(int32_t));
  }
  return PCCB200_OK;
}

// one attribute (the reference-shaped call)
template<class Exec>
int
raht_run(Exec& ex, const pccb200_raht_params& pp, const pccb200_qpset& qs,
         bool forward, const int64_t* keys, int32_t* attrs, const int32_t* qpo,
         int32_t* coef, int64_t coefStride, int A, int N)
{
  RahtSetIO io{&qs, A, coef, coefStride};
  return raht_run_sets(ex, pp, 1, &io, forward, keys, attrs, qpo, N);
}

}  // namespace pccb200
