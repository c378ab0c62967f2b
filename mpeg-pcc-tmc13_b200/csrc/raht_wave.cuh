// raht_wave.cuh — wavefront schedule of the top-down block transform
// (device only).
//
// Sub-node prediction (tmc3/RAHT.cpp:370-415) makes a block wait for the
// earlier neighbour blocks whose children it reads.  Claimed in Morton order,
// the members of a chain are all claimed at about the same time and their
// warps sit on them until the chain has been worked off.  Without the
// encoder's RDOQ (decoder; integer Haar) those are the only dependencies
// inside a stage, they follow from geometry alone, and the blocks can be
// claimed in dependency-level ("wavefront") order instead, so that a block is
// normally ready when a warp takes it.  With RDOQ the zero-run look-back
// (RAHT.cpp:1154,1576-1670) follows coding order and may reach arbitrarily far
// back: coding order stays the ticket order there (a wavefront order with
// bounded waits and restarts was measured far slower).
// The schedule, computed before any attribute value is read:
//
//   1. geometry of every stage (top-down, fully parallel kernels): qp
//      descent + neighbour counts of single-child blocks (PrepFn, mode 1),
//      worklist of the transforming blocks, the 18 neighbour searches and the
//      same-stage dependency mask of each (k_block_geom);
//   2. (no RDOQ) dependency level of every block, all stages in one launch
//      (k_block_levels): 1 + max level of the earlier neighbour blocks whose
//      children it reads;
//   3. (no RDOQ) one stable radix sort of all rows by (stage, level);
//   4. the stages, coarse to fine: reconstruction slots armed, single-child
//      blocks passed through (PrepFn, mode 2), k_block_warp over the worklist
//      in schedule order.
//
// Steps 1-3 read no attribute value: they are the same for every attribute
// coded on the same positions.
#pragma once

#include "morton_sort.cuh"
#include "raht_pipeline.cuh"

namespace pccb200 {

constexpr int kMaxWaveSegs = 24;   // descent steps below the root (<= 21)

struct LevelArgs {
  int numSeg;                   // segments 1..numSeg
  int rowOff[kMaxWaveSegs + 2]; // rowOff[d]; rowOff[numSeg + 1] = number of rows
  const int* cnt;               // cnt[d]: transforming blocks of segment d
  const int32_t* wl;            // row -> block index (first cnt[d] rows of a segment)
  const int32_t* geom;          // kGeomStride ints per transforming block, segment d at geomOff[d]
  int geomOff[kMaxWaveSegs + 2];
  int* lv;                      // per (segment, block index): dependency level, 0 = not known yet
  int64_t* key;                 // per row: segment << 16 | level (0xffff: unused row)
  int32_t* val;                 // per row: the row itself
};

// qp descent of the root block (the root block's kernel repeats it)
struct RootQpFn {
  Stage S;
  PCC_HD void operator()(int64_t) const { descend_qps(S, 0, S.n, nullptr); }
};

struct FillI32 {
  int32_t* p;
  int32_t v;
  PCC_HD void operator()(int64_t i) const { p[i] = v; }
};

// One thread per row, 32 consecutive rows per ticket, rows in coding order:
// everything a row waits for has a lower row number, hence a ticket that has
// been claimed.  The loop is uniform over the warp (a lane never spins while
// another lane of its warp could be the one it is waiting for).
__global__ void __launch_bounds__(256)
k_block_levels(const LevelArgs a, unsigned long long* ticket)
{
  const int lane = threadIdx.x & 31;
  const long long numRows = a.rowOff[a.numSeg + 1];
  for (;;) {
    unsigned long long base = 0;
    if (lane == 0)
      base = atomicAdd(ticket, 32ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base >= (unsigned long long)numRows)
      return;
    const long long row = (long long)base + lane;
    int d = 1, off = 0, t = 0, p = 0;
    bool active = false;
    if (row < numRows) {
      while (d < a.numSeg && row >= a.rowOff[d + 1])
        d++;
      off = a.rowOff[d];
      t = int(row) - off;
      active = t < a.cnt[d];
      a.val[row] = int32_t(row);
      if (!active)
        a.key[row] = (int64_t(d) << 16) | 0xffff;
    }
    uint32_t depMask = 0;
    int q[12];
#pragma unroll
    for (int i = 0; i < 12; i++)
      q[i] = 0;
    if (active) {
      p = a.wl[row];
      const int32_t* g = a.geom + (size_t(a.geomOff[d]) + t) * kGeomStride;
      depMask = (uint32_t(g[19]) >> 8) & 0xfffu;
#pragma unroll
      for (int i = 0; i < 12; i++)
        if ((depMask >> i) & 1)
          q[i] = g[7 + i];
    }
    bool done = !active;
    while (__any_sync(0xffffffffu, !done)) {
      bool progress = false;
      if (!done) {
        int m = 0;
        bool ready = true;
#pragma unroll
        for (int i = 0; i < 12; i++)
          if ((depMask >> i) & 1) {
            const int v = ld_relaxed_i32(&a.lv[off + q[i]]);
            if (!v)
              ready = false;
            else
              m = v > m ? v : m;
          }
        if (ready) {
          m++;
          st_relaxed_i32(&a.lv[off + p], m);
          a.key[row] = (int64_t(d) << 16) | (m < 0xfffe ? m : 0xfffe);
          done = true;
          progress = true;
        }
      }
      if (!__any_sync(0xffffffffu, progress))
        __nanosleep(40);
    }
  }
}

template<>
struct WaveDescent<DeviceExec> {
  static constexpr bool available = true;

  static bool enabled(const RahtConfig& cfg)
  {
    // AC-coefficient qp offsets in the encoder keep the exact-counter protocol
    // of the thread-per-block body (see DeviceExec::block_stage)
    if (cfg.isEncoder && !cfg.haar && cfg.numAcLayers > 0)
      return false;
    return true;
  }

  // Everything one unit's descent needs between its preparation (geometry,
  // schedule: steps 1-3) and its stage launches (step 4).  Kept so that the
  // stage launches of several units can be issued together (run_gang).
  // stages[0] = leaves ... stages.back() = children of the root block;
  // rt: the attributes coded in this pass (cfg.A = all their components).
  struct Job {
    RahtConfig cfg;
    int numSets = 0;
    RahtSetRt rt[kMaxSets];
    std::vector<Stage> stages;
    int top = 0;
    bool rdoq = false;
    std::vector<WarpBlockArgs> args;   // one per descent step, [0] = root block
    int rowOff[kMaxWaveSegs + 2] = {};
    int blocks[kMaxWaveSegs + 2] = {};  // transforming blocks of every step
    const int32_t* order = nullptr;
    int* cntRoot = nullptr;
    unsigned long long* tickets = nullptr;
    TzRegion* dRegions[kMaxSets] = {nullptr, nullptr};
  };

  // The stage launches of prepared units, step by step: launch d carries
  // descent step d of every unit that has one (units are independent; a step
  // needs only the previous step of its own unit).  A step of one unit runs
  // k_block_warp with the unit's arguments as its kernel parameter; a step of
  // several runs k_block_warp_gang over a table of their arguments.
  static void run_gang(DeviceExec& ex, Job* const* jobs, int numJobs)
  {
    int maxTop = -1;
    for (int u = 0; u < numJobs; u++)
      maxTop = jobs[u]->top > maxTop ? jobs[u]->top : maxTop;
    ex.phase(kPhaseBlock);
    std::vector<GangEntry> tab;
    for (int d = 0; d <= maxTop; d++) {
      tab.clear();
      int maxBlocks = 1;
      for (int u = 0; u < numJobs; u++) {
        Job& job = *jobs[u];
        if (d > job.top)
          continue;
        const int nBlocks = stage_prep(ex, job, d);
        maxBlocks = nBlocks > maxBlocks ? nBlocks : maxBlocks;
        tab.push_back(GangEntry{job.args[d], job.tickets + d});
      }
      const int units = int(tab.size());
      GangEntry* dTab = nullptr;
      if (units > 1) {
        dTab = ex.alloc<GangEntry>(tab.size());
        ex.upload(dTab, tab.data(), tab.size() * sizeof(GangEntry));
      }
      // the lane's share of the machine, divided among the units of the gang
      int64_t perUnit = ex.block_grid(int64_t(1) << 40) / units;
      const int64_t useful = (int64_t(maxBlocks) + kWarpBlockThreads / 32 - 1) / (kWarpBlockThreads / 32);
      perUnit = perUnit > useful ? useful : perUnit;
      const char* ec = getenv("PCCB200_GANG_CTAS");  // A/B: CTAs per unit (read per call)
      if (ec && atoi(ec) > 0 && perUnit > atoi(ec))
        perUnit = atoi(ec);
      perUnit = perUnit < 1 ? 1 : perUnit;
      // the variant every unit of the launch can run (raht_block_warp.cuh)
      BlockVariant variant = block_variant(tab[0].a);
      for (int u = 1; u < units; u++)
        if (block_variant(tab[u].a) != variant)
          variant = kBlockGeneric;
      {
        DeviceExec::Scope sc(ex);
        if (variant == kBlockRdoq2)
          launch_blocks<kBlockRdoq2>(ex, tab, dTab, perUnit);
        else if (variant == kBlockRdoq1)
          launch_blocks<kBlockRdoq1>(ex, tab, dTab, perUnit);
        else
          launch_blocks<kBlockGeneric>(ex, tab, dTab, perUnit);
        g_launchCount++;
      }
      PCC_CUDA_CHECK(cudaGetLastError());
    }
  }

  template<BlockVariant V>
  static void launch_blocks(DeviceExec& ex, const std::vector<GangEntry>& tab, const GangEntry* dTab,
                            int64_t perUnit)
  {
    const int units = int(tab.size());
    if (units == 1)
      k_block_warp<V><<<unsigned(perUnit), kWarpBlockThreads, 0, ex.stream>>>(tab[0].a, tab[0].ticket);
    else
      k_block_warp_gang<V><<<unsigned(perUnit * units), kWarpBlockThreads, 0, ex.stream>>>(dTab, units);
  }

  // steps 1-3 (nothing here reads an attribute value)
  static void prepare(DeviceExec& ex, const RahtConfig& cfg, int numSets, const RahtSetRt* rt,
                      const std::vector<Stage>& stages, Job& job)
  {
    const int top = int(stages.size()) - 1;
    const bool rdoq = cfg.isEncoder && !cfg.haar;
    job.cfg = cfg;
    job.numSets = numSets;
    for (int s = 0; s < numSets; s++)
      job.rt[s] = rt[s];
    job.stages = stages;
    job.top = top;
    job.rdoq = rdoq;
    const char* ep = getenv("PCCB200_POLL_NS");  // A/B knob, read per call
    const int pollNs = ep ? atoi(ep) : 32;
    const bool wave = cfg.predictionEnabled && cfg.subnode && !rdoq;

    //-- row space: one segment per descent step below the root
    LevelArgs la = {};
    la.numSeg = top;
    int64_t numRows = 0;
    for (int d = 1; d <= top; d++) {
      la.rowOff[d] = int(numRows);
      numRows += stages[top - d + 1].n;
    }
    la.rowOff[top + 1] = int(numRows);
    la.rowOff[0] = 0;
    for (int d = 0; d <= top + 1; d++)
      job.rowOff[d] = la.rowOff[d];

    int32_t* wl = ex.alloc<int32_t>(size_t(numRows));
    int* cnt = ex.alloc<int>(top + 2);  // [0]: root step, [d]: step d
    // zeroed in one go: the ticket word of every step, the levels
    const size_t zInts = size_t(top + 2) * 2 + (wave ? size_t(numRows) : 0);
    int* zero = ex.alloc<int>(zInts);
    ex.zero(zero, zInts * sizeof(int));
    unsigned long long* tickets = reinterpret_cast<unsigned long long*>(zero);
    int* lv = zero + size_t(top + 2) * 2;
    job.tickets = tickets;

    //-- 0. worklists of all steps (they follow from the tree alone); their sizes
    //   go to the host (one read-back) so that the neighbour tables -- 80 bytes
    //   per transforming block, the largest item of a unit's workspace -- are
    //   allocated for the blocks that transform (a third of all blocks on the
    //   bench frame), not for every block
    ex.phase(kPhaseGeom);
    int* cntRoot = cnt;  // cnt[0]: the root step has one block
    job.cntRoot = cntRoot;
    {
      int one = 1;
      ex.upload(cntRoot, &one, sizeof(int));
    }
    for (int d = 1; d <= top; d++)
      ex.compact(stages[top - d + 1].n, MultiChildPred{stages[top - d + 1].first},
                 WorklistEmit{wl + la.rowOff[d]}, cnt + d);
    int hostCnt[kMaxWaveSegs + 2] = {};
    int32_t* geom = nullptr;
    la.geomOff[0] = 0;
    if (top >= 1)
      ex.download(hostCnt, cnt, size_t(top + 1) * sizeof(int));
    hostCnt[0] = 1;
    for (int d = 0; d <= top; d++)
      job.blocks[d] = hostCnt[d];
    if (cfg.predictionEnabled) {
      int64_t total = 0;
      for (int d = 1; d <= top; d++) {
        la.geomOff[d] = int(total);
        total += hostCnt[d];
      }
      la.geomOff[top + 1] = int(total);
      geom = ex.alloc<int32_t>(size_t(total) * kGeomStride);
    }

    //-- 1. geometry, top-down
    ex.foreach(stages[top].n, FillI32{stages[top].nn, 19});
    if (cfg.hasQp)
      ex.foreach(1, RootQpFn{stages[top]});
    int64_t abA, abB;
    raht_ab(1, 1, abA, abB);
    std::vector<WarpBlockArgs>& args = job.args;
    args.assign(top + 1, WarpBlockArgs{});
    for (int d = 0; d <= top; d++) {
      WarpBlockArgs& a = args[d];
      a.cfg = cfg;
      a.numSets = numSets;
      for (int s = 0; s < numSets; s++) {
        AttrSet& st = a.set[s];
        st.A = rt[s].A;
        st.base = rt[s].base;
        st.maxQp = rt[s].maxQp;
        st.fixedPointQpOffset = rt[s].fixedPointQpOffset;
        st.numAcLayers = rt[s].numAcLayers;
        st.qt = rt[s].qt;
        st.coef = rt[s].coef;
        st.coefStride = rt[s].coefStride;
      }
      a.ab11a = abA;
      a.ab11b = abB;
      a.pollNs = pollNs;
    }
    for (int d = 1; d <= top; d++) {
      const int si = top - d;
      const Stage& S = stages[si];
      const Stage& P = stages[si + 1];
      const int nBlocks = P.n;
      PrepFn prep{cfg, S, P, cfg.predictionEnabled, nullptr, 1};
      if (cfg.hasQp || cfg.predictionEnabled)
        ex.foreach(nBlocks, prep);
      WarpBlockArgs& a = args[d];
      a.S = S;
      a.P = P;
      a.coefBase = P.n;
      a.predInLvl = cfg.predictionEnabled;
      a.worklist = wl + la.rowOff[d];
      a.geom = geom ? geom + size_t(la.geomOff[d]) * kGeomStride : nullptr;
      a.count = cnt + d;
      if (cfg.predictionEnabled && hostCnt[d] > 0) {
        DeviceExec::Scope sc(ex);
        k_block_geom<<<unsigned((int64_t(hostCnt[d]) * 32 + 255) / 256), 256, 0, ex.stream>>>(a);
        g_launchCount++;
      }
    }

    //-- 2 + 3. dependency levels, wavefront order
    job.order = nullptr;
    if (wave && numRows > 0) {
      ex.phase(kPhaseOrder);
      int64_t* keyA = ex.alloc<int64_t>(size_t(numRows));
      int64_t* keyB = ex.alloc<int64_t>(size_t(numRows));
      int32_t* valA = ex.alloc<int32_t>(size_t(numRows));
      int32_t* valB = ex.alloc<int32_t>(size_t(numRows));
      la.cnt = cnt;
      la.wl = wl;
      la.geom = geom;
      la.lv = lv;
      la.key = keyA;
      la.val = valA;
      {
        DeviceExec::Scope sc(ex);
        int64_t blocks = (numRows + 255) / 256;
        const int64_t cap = int64_t(ex.numSMs) * 8;
        k_block_levels<<<unsigned(blocks > cap ? cap : blocks), 256, 0, ex.stream>>>(
          la, tickets + top + 1);
        g_launchCount++;
      }
      int64_t* kres;
      int32_t* vres;
      device_radix_sort_pairs(ex, keyA, valA, keyB, valB, numRows, 3, &kres, &vres);
      job.order = vres;
    }

    // zero-run state words: one region of (blocks + 1) words per descent step
    // and attribute, all zeroed ("nothing published") in one go; the table of
    // regions (for the walk across steps) is uploaded once
    if (rdoq) {
      int64_t stateOff[kMaxWaveSegs + 3];
      stateOff[0] = 0;
      stateOff[1] = 2;
      for (int d = 1; d <= top; d++)
        stateOff[d + 1] = stateOff[d] + stages[top - d + 1].n + 1;
      const size_t words = size_t(stateOff[top + 1]);
      unsigned long long* state = ex.alloc<unsigned long long>(words * numSets);
      ex.zero(state, words * numSets * sizeof(unsigned long long));
      for (int s = 0; s < numSets; s++) {
        TzRegion hr[kMaxWaveSegs + 2];
        for (int d = 0; d <= top; d++) {
          hr[d].state = state + words * s + stateOff[d];
          hr[d].count = d == 0 ? cntRoot : cnt + d;
          args[d].set[s].state = hr[d].state;
        }
        job.dRegions[s] = ex.alloc<TzRegion>(kMaxWaveSegs + 2);
        ex.upload(job.dRegions[s], hr, sizeof(TzRegion) * (top + 1));
        for (int d = 0; d <= top; d++)
          args[d].set[s].regions = job.dRegions[s];
      }
    }
    PCC_CUDA_CHECK(cudaGetLastError());
  }

  //-- 4. what precedes the block kernel of descent step d: reconstruction
  //   slots armed, single-child blocks passed through (they read the previous
  //   step's results).  Returns the number of blocks the kernel will run.
  static int stage_prep(DeviceExec& ex, Job& job, int d)
  {
    const RahtConfig& cfg = job.cfg;
    const int top = job.top;
    const int si = top - d;
    const Stage& S = job.stages[si];
    WarpBlockArgs& a = job.args[d];
    ex.fill(S.rec, 0x80, size_t(S.n) * cfg.A * sizeof(int64_t));
    int nBlocks = 1;
    if (d == 0) {
      a.S = S;
      a.P = Stage{};
      a.P.n = 0;
      a.coefBase = 0;
      a.predInLvl = 0;
      a.worklist = nullptr;
      a.geom = nullptr;
      a.count = job.cntRoot;
    } else {
      const Stage& P = job.stages[si + 1];
      nBlocks = P.n;
      ex.foreach(nBlocks, PrepFn{cfg, S, P, cfg.predictionEnabled, nullptr, 2});
      a.order = job.order ? job.order + job.rowOff[d] : nullptr;
      a.orderBase = job.rowOff[d];
    }
    a.stageIdx = d;
    for (int s = 0; s < job.numSets; s++) {
      AttrSet& st = a.set[s];
      st.qpLayer = d + 1 < job.rt[s].numLayers ? d + 1 : job.rt[s].numLayers - 1;
      st.acLayer = d;
    }
    return job.blocks[d];
  }
};

}  // namespace pccb200
