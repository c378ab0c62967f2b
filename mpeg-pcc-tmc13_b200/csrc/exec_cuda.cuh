// exec_cuda.cuh — the CUDA executor: turns the per-item bodies of
// raht_core.cuh into kernel launches on one stream of one GPU.
//
//   foreach  : grid-stride kernel, grid sized in multiples of the SM count
//   ordered  : block-level dataflow kernel.  CTAs claim chunks of the index
//              space in ascending order through a global ticket, so every
//              index below a running CTA's chunk is owned by a CTA that is
//              already running: an item may spin on flags published by any
//              lower index without risk of deadlock, whatever the residency.
//   compact  : three-kernel stream compaction (tile counts, scan of the tile
//              counts, in-tile scan + emit); ranks are exact and ordered.
//   subsample_distance : warp-per-cell dataflow over the cells of a level
//              (lod_subsample_warp.cuh), wavefront order for large levels.
//   block_stage : one RAHT stage with the thread-per-block body; the CUDA
//              descent is otherwise WaveDescent's (raht_wave.cuh).
//
// Workspace comes from a per-context arena (one cudaMalloc in steady state).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "pcc_attr_b200.h"
#include <stdio.h>

#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "lod_subsample_warp.cuh"
#include "raht_block_warp.cuh"

namespace pccb200 {

extern std::atomic<uint64_t> g_launchCount;

struct CudaError {
  cudaError_t code;
  const char* what;
};

#define PCC_CUDA_CHECK(expr)                                   \
  do {                                                         \
    cudaError_t _e = (expr);                                   \
    if (_e != cudaSuccess)                                     \
      throw ::pccb200::CudaError{_e, #expr};                   \
  } while (0)

//----------------------------------------------------------------------------

class Arena {
public:
  ~Arena() { release(); }

  // Chunks are kept from call to call and filled in order; a call that needs
  // more gets a new chunk (cudaMalloc does not disturb running kernels).
  void* alloc(size_t bytes)
  {
    bytes = (bytes + 255) & ~size_t(255);
    while (cur_ < chunks_.size() && used_ + bytes > chunks_[cur_].size) {
      cur_++;
      used_ = 0;
    }
    if (cur_ == chunks_.size()) {
      size_t want = bytes > nextSize_ ? bytes : nextSize_;
      void* p = nullptr;
      PCC_CUDA_CHECK(cudaMalloc(&p, want));
      chunks_.push_back({p, want});
      used_ = 0;
    }
    void* r = static_cast<char*>(chunks_[cur_].ptr) + used_;
    used_ += bytes;
    high_ += bytes;
    return r;
  }

  // Start of a call.  mayFree: no other call is in flight, so the chunks may
  // be folded into one big enough for the largest call seen so far (cudaFree
  // synchronises the device: it would stall the dataflow kernels of the other
  // lanes in the middle of their polling, so it is never done under load).
  void reset(bool mayFree)
  {
    if (high_ > peak_)
      peak_ = high_;
    if (mayFree
        && (chunks_.size() > 1 || (chunks_.size() == 1 && chunks_[0].size < peak_))) {
      release();
    }
    if (chunks_.empty() && peak_) {
      void* p = nullptr;
      size_t want = peak_ + (peak_ >> 3) + (1 << 20);
      PCC_CUDA_CHECK(cudaMalloc(&p, want));
      chunks_.push_back({p, want});
    }
    cur_ = 0;
    used_ = 0;
    high_ = 0;
  }

  void release()
  {
    for (auto& c : chunks_)
      cudaFree(c.ptr);
    chunks_.clear();
    cur_ = 0;
    used_ = 0;
  }

private:
  struct Chunk {
    void* ptr;
    size_t size;
  };
  std::vector<Chunk> chunks_;
  size_t cur_ = 0;
  size_t used_ = 0;
  size_t high_ = 0;
  size_t peak_ = 0;
  size_t nextSize_ = size_t(64) << 20;
};

//----------------------------------------------------------------------------
// kernels

template<class F>
__global__ void __launch_bounds__(256)
k_foreach(F f, int64_t n)
{
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x)
    f(i);
}

constexpr int kOrderedThreads = 128;

template<class F>
__global__ void __launch_bounds__(kOrderedThreads)
k_ordered(F f, int64_t n, unsigned long long* ticket)
{
  __shared__ unsigned long long sBase;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nWarps = kOrderedThreads / 32;
  for (;;) {
    if (threadIdx.x == 0)
      sBase = atomicAdd(ticket, (unsigned long long)kOrderedThreads);
    __syncthreads();
    const int64_t base = int64_t(sBase);
    __syncthreads();
    if (base >= n)
      return;
    // lanes of one warp take items nWarps apart so that directly adjacent
    // items (the commonest dependency) sit in different warps
    const int64_t i = base + lane * nWarps + warp;
    if (i < n)
      f(i);
  }
}

// Warp-uniform dataflow over a gang of chains: CTA b serves chain
// items[b % numItems] (as k_block_warp_gang serves units).  Each warp claims
// 32 consecutive tickets of its chain (item.ticket, item.size() of them);
// item(t) returns false while ticket t waits for a lower ticket of the same
// chain.  Lanes of a warp never spin against each other: the ready ones run,
// and the warp repeats (the k_cell_levels pattern).  Lower tickets are held
// by running warps, so any grid is free of deadlock.
template<class F>
__global__ void __launch_bounds__(256)
k_warp_flow(const F* __restrict__ items, int numItems)
{
  const F& f = items[blockIdx.x % numItems];
  const int64_t n = f.size();
  const int lane = threadIdx.x & 31;
  for (;;) {
    unsigned long long base = 0;
    if (lane == 0)
      base = atomicAdd(f.ticket, 32ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base >= (unsigned long long)n)
      return;
    const int64_t t = int64_t(base) + lane;
    bool done = t >= n;
    while (__any_sync(0xffffffffu, !done)) {
      bool progress = false;
      if (!done && f(t))
        done = progress = true;
      if (!__any_sync(0xffffffffu, progress))
        __nanosleep(40);
    }
  }
}

constexpr int kTileThreads = 256;
constexpr int kTileItems = 8;
constexpr int kTile = kTileThreads * kTileItems;

template<class P>
__global__ void __launch_bounds__(kTileThreads)
k_tile_count(P pred, int64_t n, int* tileCount)
{
  const int64_t base = int64_t(blockIdx.x) * kTile + threadIdx.x * kTileItems;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kTileItems; j++)
    if (base + j < n && pred(base + j))
      c++;
  // block reduce
  __shared__ int sWarp[kTileThreads / 32];
#pragma unroll
  for (int o = 16; o; o >>= 1)
    c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0)
    sWarp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kTileThreads / 32; w++)
      t += sWarp[w];
    tileCount[blockIdx.x] = t;
  }
}

// exclusive scan of the tile counts by a single CTA (tile counts are few:
// n / 2048)
__global__ void __launch_bounds__(1024)
k_scan_tiles(int* tileCount, int numTiles, int* total)
{
  __shared__ int sWarp[32];
  __shared__ int sCarry;
  if (threadIdx.x == 0)
    sCarry = 0;
  __syncthreads();
  for (int base = 0; base < numTiles; base += 1024) {
    int i = base + threadIdx.x;
    int v = i < numTiles ? tileCount[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o)
        x += y;
    }
    if ((threadIdx.x & 31) == 31)
      sWarp[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int s = sWarp[threadIdx.x];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, s, o);
        if (threadIdx.x >= o)
          s += y;
      }
      sWarp[threadIdx.x] = s;
    }
    __syncthreads();
    int warpOff = (threadIdx.x >> 5) ? sWarp[(threadIdx.x >> 5) - 1] : 0;
    int carry = sCarry;
    if (i < numTiles)
      tileCount[i] = carry + warpOff + x - v;
    __syncthreads();
    if (threadIdx.x == 1023)
      sCarry = carry + warpOff + x;
    __syncthreads();
  }
  if (total && threadIdx.x == 0)
    *total = sCarry;
}

template<class P, class E>
__global__ void __launch_bounds__(kTileThreads)
k_tile_emit(P pred, E emit, int64_t n, const int* tileOffset)
{
  const int64_t base = int64_t(blockIdx.x) * kTile + threadIdx.x * kTileItems;
  unsigned flags = 0;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kTileItems; j++)
    if (base + j < n && pred(base + j)) {
      flags |= 1u << j;
      c++;
    }
  // exclusive scan of c over the CTA
  __shared__ int sWarp[kTileThreads / 32];
  int x = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) >= o)
      x += y;
  }
  if ((threadIdx.x & 31) == 31)
    sWarp[threadIdx.x >> 5] = x;
  __syncthreads();
  int warpOff = 0;
  for (int w = 0; w < (threadIdx.x >> 5); w++)
    warpOff += sWarp[w];
  int64_t rank = int64_t(tileOffset[blockIdx.x]) + warpOff + x - c;
#pragma unroll
  for (int j = 0; j < kTileItems; j++)
    if ((flags >> j) & 1)
      emit(rank++, base + j);
}

//----------------------------------------------------------------------------

// optional per-phase timing: one event pair per launch, resolved after the
// call's final synchronisation
struct Profiler {
  bool enabled = false;
  double ms[PCCB200_NUM_PHASES] = {};
  uint64_t launches[PCCB200_NUM_PHASES] = {};
  struct Pending {
    int phase;
    cudaEvent_t a, b;
  };
  std::vector<Pending> pending;
  std::vector<cudaEvent_t> pool;

  cudaEvent_t get()
  {
    if (!pool.empty()) {
      cudaEvent_t e = pool.back();
      pool.pop_back();
      return e;
    }
    cudaEvent_t e;
    PCC_CUDA_CHECK(cudaEventCreate(&e));
    return e;
  }
  void resolve()
  {
    static const bool debug = getenv("PCCB200_DEBUG") != nullptr;
    if (debug && !pending.empty())
      fprintf(stderr, "[pccb200] block-transform launches (ms):");
    for (auto& p : pending) {
      float t = 0;
      if (cudaEventElapsedTime(&t, p.a, p.b) == cudaSuccess) {
        ms[p.phase] += t;
        launches[p.phase]++;
        if (debug && p.phase == 2)
          fprintf(stderr, " %.3f", t);
      }
      pool.push_back(p.a);
      pool.push_back(p.b);
    }
    if (debug && !pending.empty())
      fprintf(stderr, "\n");
    pending.clear();
  }
};

enum Phase {
  kPhaseSort = 0, kPhaseTree, kPhaseBlock, kPhaseTail, kPhaseGather, kPhaseLift, kPhaseGeom,
  kPhaseOrder
};

struct DeviceExec {
  cudaStream_t stream = nullptr;
  Arena* arena = nullptr;
  int numSMs = 132;
  unsigned long long* ticket = nullptr;  // device word for ordered launches
  Profiler* prof = nullptr;
  int curPhase = 0;
  const std::atomic<int>* activeCalls = nullptr;  // calls in flight (all lanes)

  void phase(int p) { curPhase = p; }

  // brackets one launch (or a short group of launches) with events
  struct Scope {
    DeviceExec& ex;
    cudaEvent_t a = nullptr, b = nullptr;
    explicit Scope(DeviceExec& e) : ex(e)
    {
      if (ex.prof && ex.prof->enabled) {
        a = ex.prof->get();
        b = ex.prof->get();
        cudaEventRecord(a, ex.stream);
      }
    }
    ~Scope()
    {
      if (a) {
        cudaEventRecord(b, ex.stream);
        ex.prof->pending.push_back({ex.curPhase, a, b});
      }
    }
  };

  template<class T>
  T* alloc(size_t n)
  {
    return static_cast<T*>(arena->alloc((n ? n : 1) * sizeof(T)));
  }

  void zero(void* p, size_t bytes)
  {
    PCC_CUDA_CHECK(cudaMemsetAsync(p, 0, bytes, stream));
  }

  void fill(void* p, int byte, size_t bytes)
  {
    PCC_CUDA_CHECK(cudaMemsetAsync(p, byte, bytes, stream));
  }

  void upload(void* dst, const void* src, size_t bytes)
  {
    // small parameter blocks: the source may be a stack temporary, so the
    // copy must have completed (or been staged) when this returns.  Pageable
    // sources make cudaMemcpyAsync stage synchronously.
    PCC_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
  }

  void download(void* dst, const void* src, size_t bytes)
  {
    PCC_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream));
    PCC_CUDA_CHECK(cudaStreamSynchronize(stream));
  }

  // Morton keys + stable radix sort (defined in morton_sort.cuh)
  void morton_sort(const int32_t* xyz, int64_t n, int64_t* keys, int32_t* order);
  // in-place exclusive prefix sum (defined in morton_sort.cuh)
  void exclusive_scan(int* data, int64_t n);

  template<class F>
  void foreach(int64_t n, const F& f)
  {
    if (n <= 0)
      return;
    int64_t blocks = (n + 255) / 256;
    int64_t cap = int64_t(numSMs) * 16;
    if (blocks > cap)
      blocks = cap;
    Scope sc(*this);
    k_foreach<F><<<unsigned(blocks), 256, 0, stream>>>(f, n);
    g_launchCount++;
    PCC_CUDA_CHECK(cudaGetLastError());
  }

  template<class F>
  void ordered(int64_t n, const F& f)
  {
    if (n <= 0)
      return;
    PCC_CUDA_CHECK(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
    int perSM = 0;
    PCC_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
      &perSM, k_ordered<F>, kOrderedThreads, 0));
    if (perSM < 1)
      perSM = 1;
    int64_t blocks = (n + kOrderedThreads - 1) / kOrderedThreads;
    int64_t cap = int64_t(numSMs) * perSM;
    if (blocks > cap)
      blocks = cap;
    Scope sc(*this);
    k_ordered<F><<<unsigned(blocks), kOrderedThreads, 0, stream>>>(f, n, ticket);
    g_launchCount++;
    PCC_CUDA_CHECK(cudaGetLastError());
  }

  // One k_warp_flow launch over numItems chains: hItems on the host, dItems
  // the same in executor memory, their tickets zeroed.  The persistent grid
  // is the resident CTAs of the machine shared among the calls in flight, a
  // multiple of the number of chains, and no more than their items need.
  template<class F>
  void flow(const F* hItems, const F* dItems, int numItems)
  {
    if (numItems <= 0)
      return;
    static const int perSM = [] {
      int v = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_warp_flow<F>, 256, 0) != cudaSuccess)
        v = 0;
      return v < 1 ? 1 : v;
    }();
    int64_t cap = int64_t(numSMs) * perSM;
    const int inFlight = activeCalls ? activeCalls->load() : 1;
    if (inFlight > 1)
      cap /= inFlight;
    int64_t perChain = 1;
    for (int c = 0; c < numItems; c++) {
      const int64_t want = (hItems[c].size() + 255) / 256;
      perChain = want > perChain ? want : perChain;
    }
    int64_t fit = cap / numItems;
    if (fit < 1)
      fit = 1;
    if (perChain > fit)
      perChain = fit;
    Scope sc(*this);
    k_warp_flow<F><<<unsigned(perChain * numItems), 256, 0, stream>>>(dItems, numItems);
    g_launchCount++;
    PCC_CUDA_CHECK(cudaGetLastError());
  }

  template<class P, class E>
  void compact(int64_t n, const P& pred, const E& emit, int* total = nullptr)
  {
    if (n <= 0) {
      if (total)
        zero(total, sizeof(int));
      return;
    }
    int numTiles = int((n + kTile - 1) / kTile);
    int* tiles = alloc<int>(numTiles);
    Scope sc(*this);
    k_tile_count<P><<<numTiles, kTileThreads, 0, stream>>>(pred, n, tiles);
    k_scan_tiles<<<1, 1024, 0, stream>>>(tiles, numTiles, total);
    k_tile_emit<P, E><<<numTiles, kTileThreads, 0, stream>>>(pred, emit, n, tiles);
    g_launchCount += 3;
    PCC_CUDA_CHECK(cudaGetLastError());
  }

  // cells sorted by dependency level (defined in morton_sort.cuh: needs the radix sort)
  const int32_t* cell_wave_order(const int32_t* nb, int nCells);

  // Distance subsampling over cells in Morton order (see lod_subsample_warp.cuh)
  void subsample_distance(const SubsampleDistanceFn& fn, int nCells)
  {
    if (nCells <= 0)
      return;
    SubsampleCellsArgs a;
    a.v = fn.v;
    a.input = fn.input;
    a.cellFirst = fn.cellFirst;
    a.nCells = nCells;
    a.shiftBits0 = fn.shiftBits0;
    a.decision = fn.decision;
    a.keep = fn.keep;
    a.nb = alloc<int32_t>(size_t(nCells) * 19);
    a.decPos = alloc<int4>(size_t(nCells));
    zero(a.decPos, size_t(nCells) * sizeof(int4));
    a.order = nullptr;
    Scope sc(*this);
    const int64_t threads = int64_t(nCells) * 19;
    k_cell_neighbours<<<unsigned((threads + 255) / 256), 256, 0, stream>>>(a);
    // wavefront order for the large levels (see k_cell_levels)
    if (nCells >= 4096)
      a.order = cell_wave_order(a.nb, nCells);
    PCC_CUDA_CHECK(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
    int64_t blocks = (int64_t(nCells) + 7) / 8;
    const int inFlight = activeCalls ? activeCalls->load() : 1;
    int64_t cap = int64_t(numSMs) * 8;
    if (inFlight > 1)
      cap /= 2 * inFlight;
    if (cap < 8)
      cap = 8;
    if (blocks > cap)
      blocks = cap;
    k_subsample_cells<<<unsigned(blocks), 256, 0, stream>>>(a, ticket);
    g_launchCount += 2;
    PCC_CUDA_CHECK(cudaGetLastError());
  }


  // Persistent grid of the block kernels for a stage of nBlocks blocks: the
  // resident CTAs of the machine, shared among the calls in flight.
  int64_t block_grid(int64_t nBlocks) const
  {
    static const int perSM = [] {
      int v = 0;
      // (the generic variant: the leaner ones may fit more CTAs per SM, but more
      // resident warps per SM measured slower -- see below)
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_block_warp_gang<kBlockGeneric>,
                                                        kWarpBlockThreads, 0)
          != cudaSuccess)
        v = 0;
      return v < 1 ? 1 : v;
    }();
    const int64_t perCta = kWarpBlockThreads / 32;  // (at least one ticket per warp)
    int64_t blocks = (nBlocks + perCta - 1) / perCta;
    // calls in flight share the machine: the persistent grid of each takes
    // its part (sampled at launch time).  Together the persistent grids of the
    // calls in flight fill the machine once (measured best on the bench: 50 %
    // and 75 % were slower, and so were more resident warps per SM); the short
    // kernels of other calls (sort, tree build, PrepFn ...) get their turn as
    // CTAs retire between stages.
    const int inFlight = activeCalls ? activeCalls->load() : 1;
    int64_t cap = int64_t(numSMs) * perSM;
    // percent of the machine all calls in flight may hold (A/B knob, read per call)
    const char* es = getenv("PCCB200_BLOCK_SHARE");
    const int capShare = es ? atoi(es) : 100;
    if (inFlight > 1)
      cap = cap * capShare / (100 * inFlight);
    static const int envCap = [] {
      const char* e = getenv("PCCB200_BLOCK_GRID");
      return e ? atoi(e) : 0;
    }();
    if (envCap > 0)
      cap = envCap;
    if (cap < 8)
      cap = 8;
    return blocks > cap ? cap : blocks;
  }

  // One top-down stage with the thread-per-block body (BlockFn): the stage
  // where WaveDescent does not run, i.e. the encoder with AC-coefficient qp
  // offsets.  Those make the RDOQ decision matter even for coefficients that
  // quantise to zero, so that case keeps the exact zero-run counter protocol
  // of this body, handed from stage to stage through tzNext.
  template<class Fn>
  void block_stage(const Fn& fn, int64_t nBlocks, int* tzNext)
  {
    if (fn.P.n == 0) {
      foreach(1, fn);
    } else {
      foreach(nBlocks, PrepFn{fn.cfg, fn.S, fn.P, fn.predInLvl, fn.tz});
      ordered(nBlocks, SkipSinglesFn<Fn>{fn});
    }
    if (tzNext)
      foreach(1, TzCarryFn{fn.tz, nullptr, int(nBlocks), tzNext});
  }
};

}  // namespace pccb200
