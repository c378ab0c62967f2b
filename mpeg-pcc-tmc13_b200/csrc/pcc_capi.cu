// pcc_capi.cu — the C ABI (include/pcc_attr_b200.h) over the CUDA kernels.
//
// Every entry point: validate, stage the caller's host arrays into HBM, run
// the kernels on the context's stream, copy results back, synchronise.  No
// CPU implementation exists behind this ABI: without a usable sm_90 device
// every compute entry point returns PCCB200_ERR_NO_DEVICE.
//
// The attribute-RAHT entries (single attribute, slices, several attributes,
// batches; host or device pointers) describe their work as coding units
// (RahtUnit) and share one pipeline: code_raht chooses fused or per-attribute
// passes and deals the units to lanes, code_units codes a gang of them on one
// lane.  The attribute-lifting entries (single, slices, a level-of-detail
// handle, several attribute sets, batches; host or device pointers) share
// code_lift, one LiftUnit per lane.
// The recolouring entries (one or several attribute sets, one unit or a batch;
// host or device pointers) share code_recolour, one RecolourUnit per lane.
#include <cuda_runtime.h>

#include <stdlib.h>

#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "exec_cuda.cuh"
#include "lifting.cuh"
#include "lift_pipeline.cuh"
#include "lod_pipeline.cuh"
#include "pred_pipeline.cuh"
#include "morton_sort.cuh"
#include "pcc_attr_b200.h"
#include "raht_pipeline.cuh"
#include "raht_wave.cuh"
#include "spherical.cuh"
#include "symbols.cuh"
#include "dist2.cuh"
#include "recolour.cuh"

// behind a pccb200_lod_handle (the header declares the type at global scope)
struct pccb200_lod_handle_s {
  int device;
  pccb200_lod_params params;
  pccb200::LodState st;
  void* block = nullptr;  // one device allocation behind preds / idx / qw
  // the lifting quantisation weights are computed by the first lifting call on
  // the handle (a handle made for the predicting transform never needs them)
  std::mutex qwMu;
  bool qwReady = false;
  // made by pccb200_lod_import from the caller's levels of detail: never
  // reusable, and with scalable set its weights are the scalable ones of scal
  bool imported = false;
  bool scalable = false;
  pccb200_lod_scalable scal = {};
};

namespace pccb200 {

std::atomic<uint64_t> g_launchCount{0};

namespace {

thread_local std::string t_lastError;

// One lane = one CUDA stream with its own workspace arena, ticket word and
// event pool.  Every API call runs on one lane; calls from different host
// threads (slices, attributes, frames are independent work units,
// tmc3/encoder.cpp:545-568,1052) run on different lanes and overlap on the
// device.  Lanes are created on demand up to kMaxLanes.
struct Lane {
  cudaStream_t stream = nullptr;
  Arena arena;
  unsigned long long* ticket = nullptr;
  cudaEvent_t tail = nullptr;  // "everything queued so far" marker (pccb200_time_end)
  Profiler prof;
  bool busy = false;
};

constexpr int kMaxLanes = 32;

struct Context {
  std::mutex mu;
  std::condition_variable cv;
  int device = 0;
  bool ready = false;
  int numSMs = 0;
  std::atomic<int> active{0};
  std::vector<std::unique_ptr<Lane>> lanes;
  // profiling totals over all lanes
  bool profEnabled = false;
  double profMs[PCCB200_NUM_PHASES] = {};
  uint64_t profLaunches[PCCB200_NUM_PHASES] = {};
  // whole-device timing (pccb200_time_begin / _end)
  cudaStream_t timeStream = nullptr;
  cudaEvent_t timeBegin = nullptr, timeEnd = nullptr;
};

Context&
ctx()
{
  static Context c;
  return c;
}

int
fail(int code, const std::string& msg)
{
  t_lastError = msg;
  return code;
}

// returns PCCB200_OK or an error; must hold c.mu
int
ensure_ready(Context& c)
{
  if (c.ready)
    return PCCB200_OK;
  // (one hardware queue per lane needs CUDA_DEVICE_MAX_CONNECTIONS=32 in the
  // application's environment before its CUDA context exists: see the header)
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    cudaGetLastError();
    return fail(PCCB200_ERR_NO_DEVICE,
                std::string("no CUDA device: ") + cudaGetErrorString(e));
  }
  if (c.device >= count)
    return fail(PCCB200_ERR_NO_DEVICE, "device index out of range");
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, c.device);
  if (e != cudaSuccess)
    return fail(PCCB200_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return fail(PCCB200_ERR_NO_DEVICE,
                std::string("kernels are built for sm_90a only; device is ") + prop.name);
  e = cudaSetDevice(c.device);
  if (e != cudaSuccess)
    return fail(PCCB200_ERR_CUDA, cudaGetErrorString(e));
  c.numSMs = prop.multiProcessorCount;
  c.ready = true;
  return PCCB200_OK;
}

// must hold c.mu; creates the lane's device objects
int
make_lane(Context& c, Lane& l)
{
  cudaError_t e = cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking);
  if (e != cudaSuccess)
    return fail(PCCB200_ERR_CUDA, cudaGetErrorString(e));
  e = cudaMalloc(&l.ticket, 256);
  if (e != cudaSuccess)
    return fail(PCCB200_ERR_NOMEM, cudaGetErrorString(e));
  e = cudaEventCreateWithFlags(&l.tail, cudaEventDisableTiming);
  if (e != cudaSuccess)
    return fail(PCCB200_ERR_CUDA, cudaGetErrorString(e));
  return PCCB200_OK;
}

void
destroy_lanes(Context& c)
{
  for (auto& l : c.lanes) {
    cudaStreamSynchronize(l->stream);
    l->arena.release();
    cudaFree(l->ticket);
    if (l->tail)
      cudaEventDestroy(l->tail);
    cudaStreamDestroy(l->stream);
  }
  c.lanes.clear();
}

template<class T>
T*
to_device(DeviceExec& ex, const T* host, size_t n)
{
  T* d = ex.alloc<T>(n);
  if (n)
    PCC_CUDA_CHECK(cudaMemcpyAsync(d, host, n * sizeof(T), cudaMemcpyHostToDevice, ex.stream));
  return d;
}

template<class T>
void
to_host(DeviceExec& ex, T* host, const T* dev, size_t n)
{
  if (n)
    PCC_CUDA_CHECK(cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, ex.stream));
}

// runs body(ex) on a free lane, CUDA errors mapped to a status
template<class Body>
int
with_device(Body body)
{
  Context& c = ctx();
  Lane* lane = nullptr;
  {
    std::unique_lock<std::mutex> lock(c.mu);
    int rc = ensure_ready(c);
    if (rc != PCCB200_OK)
      return rc;
    for (;;) {
      for (auto& l : c.lanes)
        if (!l->busy) {
          lane = l.get();
          break;
        }
      if (lane)
        break;
      if (int(c.lanes.size()) < kMaxLanes) {
        cudaSetDevice(c.device);
        std::unique_ptr<Lane> l(new Lane);
        rc = make_lane(c, *l);
        if (rc != PCCB200_OK)
          return rc;
        lane = l.get();
        c.lanes.push_back(std::move(l));
        break;
      }
      c.cv.wait(lock);
    }
    lane->busy = true;
    lane->prof.enabled = c.profEnabled;
    ++c.active;
  }
  int rc;
  try {
    PCC_CUDA_CHECK(cudaSetDevice(c.device));
    lane->arena.reset(c.active.load() == 1);
    DeviceExec ex;
    ex.stream = lane->stream;
    ex.arena = &lane->arena;
    ex.numSMs = c.numSMs;
    ex.ticket = lane->ticket;
    ex.prof = &lane->prof;
    ex.activeCalls = &c.active;
    rc = body(ex);
    PCC_CUDA_CHECK(cudaStreamSynchronize(lane->stream));
    lane->prof.resolve();
    if (rc != PCCB200_OK && t_lastError.empty())
      t_lastError = "invalid argument";
  } catch (const CudaError& e) {
    cudaGetLastError();
    rc = fail(e.code == cudaErrorMemoryAllocation ? PCCB200_ERR_NOMEM : PCCB200_ERR_CUDA,
              std::string(e.what) + ": " + cudaGetErrorString(e.code));
  } catch (const std::bad_alloc&) {
    rc = fail(PCCB200_ERR_NOMEM, "host allocation failed");
  } catch (const std::exception& e) {
    rc = fail(PCCB200_ERR_CUDA, std::string("internal error: ") + e.what());
  } catch (...) {
    rc = fail(PCCB200_ERR_CUDA, "internal error");
  }
  if (rc != PCCB200_OK)  // nothing of a failed call may still be running on the lane
    cudaStreamSynchronize(lane->stream);
  {
    std::lock_guard<std::mutex> lock(c.mu);
    for (int i = 0; i < PCCB200_NUM_PHASES; i++) {
      c.profMs[i] += lane->prof.ms[i];
      c.profLaunches[i] += lane->prof.launches[i];
      lane->prof.ms[i] = 0;
      lane->prof.launches[i] = 0;
    }
    lane->busy = false;
    c.active--;
  }
  c.cv.notify_one();
  return rc;
}

// runs fn(i) for i in [0, n) on up to maxThreads host threads; returns the
// first non-zero status
template<class Fn>
int
parallel_for(int n, int maxThreads, Fn fn)
{
  if (n == 1 || maxThreads <= 1) {
    for (int i = 0; i < n; i++) {
      int rc = fn(i);
      if (rc)
        return rc;
    }
    return 0;
  }
  std::atomic<int> next{0}, status{0};
  std::string err;
  std::mutex errMu;
  auto worker = [&] {
    for (;;) {
      int i = next.fetch_add(1);
      if (i >= n)
        return;
      int rc;
      try {
        rc = fn(i);
      } catch (...) {  // a worker thread must not let anything escape
        rc = fail(PCCB200_ERR_CUDA, "internal error in a slice worker");
      }
      if (rc) {
        int expected = 0;
        if (status.compare_exchange_strong(expected, rc)) {
          std::lock_guard<std::mutex> g(errMu);
          err = t_lastError;
        }
      }
    }
  };
  int nt = n < maxThreads ? n : maxThreads;
  std::vector<std::thread> ts;
  for (int t = 1; t < nt; t++)
    ts.emplace_back(worker);
  worker();
  for (auto& t : ts)
    t.join();
  if (status.load())
    t_lastError = err;
  return status.load();
}

int
raht_common(bool forward, const pccb200_raht_params* params, const pccb200_qpset* qpset,
            const int32_t* qpo, const int64_t* morton, int32_t* attrs, int A, int n,
            int32_t* coeffs)
{
  if (!params || !qpset || !morton || !attrs || !coeffs || n <= 0 || A < 1 || A > 3)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    int64_t* dKeys = to_device(ex, morton, size_t(n));
    int32_t* dAttrs = forward ? to_device(ex, attrs, size_t(n) * A)
                              : ex.alloc<int32_t>(size_t(n) * A);
    int32_t* dQpo = qpo ? to_device(ex, qpo, size_t(n) * 2) : nullptr;
    int32_t* dCoef = forward ? ex.alloc<int32_t>(size_t(n) * A)
                             : to_device(ex, coeffs, size_t(n) * A);
    int rc = raht_run(ex, *params, *qpset, forward, dKeys, dAttrs, dQpo, dCoef,
                      int64_t(n), A, n);
    if (rc != PCCB200_OK)
      return fail(rc, rc == PCCB200_ERR_UNSORTED ? "morton codes not ascending"
                                                 : "invalid parameters");
    to_host(ex, attrs, dAttrs, size_t(n) * A);
    if (forward)
      to_host(ex, coeffs, dCoef, size_t(n) * A);
    return PCCB200_OK;
  });
}

// slice s of a frame is points [sliceOffsets[s], sliceOffsets[s + 1]): at
// least one slice, none empty, none over INT32_MAX points
int
check_offsets(const int64_t* sliceOffsets, int numSlices)
{
  if (!sliceOffsets || numSlices <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  for (int s = 0; s < numSlices; s++) {
    int64_t len = sliceOffsets[s + 1] - sliceOffsets[s];
    if (len <= 0 || len > INT32_MAX)
      return fail(PCCB200_ERR_INVALID_ARG, "empty or oversized slice");
  }
  return PCCB200_OK;
}

int
check_slices(const void* params, const void* qpset, const void* xyz, const void* attrs,
             const void* coeffs, int A, int bitdepth, const int64_t* sliceOffsets,
             int numSlices)
{
  if (!params || !qpset || !xyz || !attrs || !coeffs || A < 1 || A > 3 || bitdepth < 1
      || bitdepth > 16)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return check_offsets(sliceOffsets, numSlices);
}

int
check_multi(const void* params, int numSets, const pccb200_qpset* const* qpsets, const void* xyz,
            const void* const* attrs, const int32_t* A, const int32_t* bitdepth,
            const void* const* coeffs, int64_t n)
{
  if (!params || !qpsets || !xyz || !attrs || !A || !bitdepth || !coeffs || n <= 0
      || n > INT32_MAX || numSets < 1 || numSets > 2)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  int total = 0;
  for (int s = 0; s < numSets; s++) {
    if (!qpsets[s] || !attrs[s] || !coeffs[s] || A[s] < 1 || A[s] > 3 || bitdepth[s] < 1
        || bitdepth[s] > 16)
      return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad attribute description");
    total += A[s];
  }
  if (total > 4)
    return fail(PCCB200_ERR_INVALID_ARG, "more than four components in one pass");
  return PCCB200_OK;
}

// One coding unit of an attribute-RAHT call (a slice, or a whole frame): n
// points with their positions and optional point qp offsets ([n, 2]), and per
// attribute set its rows ([n, A], in and out) and coefficient planes
// (component k at coef + k * coefStride).  dev: device pointers, coded in
// place; otherwise host pointers.
struct RahtUnit {
  int n = 0;
  const int32_t* xyz = nullptr;
  const int32_t* qpo = nullptr;
  bool dev = false;
  int numSets = 0;
  const pccb200_qpset* qs[kMaxSets] = {};
  int A[kMaxSets] = {};
  int bitdepth[kMaxSets] = {};
  int32_t* attrs[kMaxSets] = {};
  int32_t* coef[kMaxSets] = {};
  int64_t coefStride[kMaxSets] = {};

  RahtUnit only(int s) const  // the same unit with set s alone
  {
    RahtUnit u = *this;
    u.numSets = 1;
    u.qs[0] = qs[s];
    u.A[0] = A[s];
    u.bitdepth[0] = bitdepth[s];
    u.attrs[0] = attrs[s];
    u.coef[0] = coef[s];
    u.coefStride[0] = coefStride[s];
    return u;
  }
};

// Codes a gang of units on one lane.  Each unit in turn is staged in, Morton
// sorted and gathered, and its tree built with the descent left prepared; the
// descents of all of them are issued together (WaveDescent::run_gang); then
// each unit's tail runs, its reconstruction is clipped and scattered back to
// input order and its results are staged out.
int
code_units(DeviceExec& ex, bool forward, const pccb200_raht_params& pp, const RahtUnit* units,
           int m)
{
  struct Staged {
    int32_t* order;
    int32_t* rows;  // [n, AT]: the components of every set, Morton order
    int AT;
    int32_t* out[kMaxSets];
    int32_t* coef[kMaxSets];
    int64_t coefStride[kMaxSets];
    RahtDeferred<DeviceExec> defer;
  };
  std::vector<Staged> st(m);
  for (int i = 0; i < m; i++) {
    const RahtUnit& u = units[i];
    Staged& w = st[i];
    const int n = u.n;
    const int32_t* dXyz = u.dev ? u.xyz : to_device(ex, u.xyz, size_t(n) * 3);
    const int32_t* dQpoIn = u.qpo && !u.dev ? to_device(ex, u.qpo, size_t(n) * 2) : u.qpo;
    const int32_t* dIn[kMaxSets] = {};
    w.AT = 0;
    for (int s = 0; s < u.numSets; s++) {
      const size_t len = size_t(n) * u.A[s];
      w.AT += u.A[s];
      if (u.dev) {  // in place: the gather reads the rows before the scatter overwrites them
        dIn[s] = w.out[s] = u.attrs[s];
        w.coef[s] = u.coef[s];
        w.coefStride[s] = u.coefStride[s];
        continue;
      }
      dIn[s] = forward ? to_device(ex, u.attrs[s], len) : nullptr;
      w.out[s] = ex.alloc<int32_t>(len);
      w.coef[s] = ex.alloc<int32_t>(len);
      w.coefStride[s] = n;
      if (!forward)
        PCC_CUDA_CHECK(cudaMemcpy2DAsync(w.coef[s], size_t(n) * sizeof(int32_t), u.coef[s],
                                         size_t(u.coefStride[s]) * sizeof(int32_t),
                                         size_t(n) * sizeof(int32_t), size_t(u.A[s]),
                                         cudaMemcpyHostToDevice, ex.stream));
    }
    int64_t* dKeys = ex.alloc<int64_t>(size_t(n));
    w.order = ex.alloc<int32_t>(size_t(n));
    w.rows = ex.alloc<int32_t>(size_t(n) * w.AT);
    int32_t* dQpo = dQpoIn ? ex.alloc<int32_t>(size_t(n) * 2) : nullptr;
    device_morton_sort(ex, dXyz, n, dKeys, w.order);
    const unsigned g = grid_for(n, ex.numSMs);
    ex.phase(kPhaseGather);
    RahtSetIO io[kMaxSets];
    for (int s = 0, base = 0; s < u.numSets; base += u.A[s], s++) {
      if (forward) {
        DeviceExec::Scope sc(ex);
        k_gather_rows_strided<<<g, 256, 0, ex.stream>>>(dIn[s], w.order, n, u.A[s], w.rows, w.AT,
                                                        base);
        g_launchCount++;
      }
      io[s] = RahtSetIO{u.qs[s], u.A[s], w.coef[s], w.coefStride[s]};
    }
    if (dQpo) {
      DeviceExec::Scope sc(ex);
      k_gather_rows_strided<<<g, 256, 0, ex.stream>>>(dQpoIn, w.order, n, 2, dQpo, 2, 0);
      g_launchCount++;
    }
    int rc = raht_run_sets(ex, pp, u.numSets, io, forward, dKeys, w.rows, dQpo, n, &w.defer);
    if (rc != PCCB200_OK)
      return fail(rc, "invalid parameters");
  }
  std::vector<WaveDescent<DeviceExec>::Job*> jobs;
  for (Staged& w : st)
    if (w.defer.pending)
      jobs.push_back(&w.defer.job);
  if (!jobs.empty())
    WaveDescent<DeviceExec>::run_gang(ex, jobs.data(), int(jobs.size()));
  for (int i = 0; i < m; i++) {
    const RahtUnit& u = units[i];
    Staged& w = st[i];
    const int n = u.n;
    if (w.defer.pending) {
      ex.phase(kPhaseTail);
      ex.foreach(w.defer.nLeaves, w.defer.tail);
    }
    const unsigned g = grid_for(n, ex.numSMs);
    ex.phase(kPhaseGather);
    for (int s = 0, base = 0; s < u.numSets; base += u.A[s], s++) {
      DeviceExec::Scope sc(ex);
      k_scatter_rows_clip_strided<<<g, 256, 0, ex.stream>>>(w.rows, w.AT, base, w.order, n, u.A[s],
                                                            (1 << u.bitdepth[s]) - 1, w.out[s]);
      g_launchCount++;
    }
    PCC_CUDA_CHECK(cudaGetLastError());
    if (u.dev)
      continue;
    for (int s = 0; s < u.numSets; s++) {
      to_host(ex, u.attrs[s], w.out[s], size_t(n) * u.A[s]);
      if (forward)
        PCC_CUDA_CHECK(cudaMemcpy2DAsync(u.coef[s], size_t(u.coefStride[s]) * sizeof(int32_t),
                                         w.coef[s], size_t(n) * sizeof(int32_t),
                                         size_t(n) * sizeof(int32_t), size_t(u.A[s]),
                                         cudaMemcpyDeviceToHost, ex.stream));
    }
  }
  return PCCB200_OK;
}

// Validated units, coded on the lanes.  A unit with several attribute sets is
// coded in one fused pass (one sort, one tree, one dependency chain) where the
// parameters have one, otherwise as one unit per set; results do not depend
// on the route.  The units are dealt to the lanes in gangs: a lane prepares
// the units of its gang in turn and then issues the top-down passes of all of
// them together, one launch per descent step.  A textured unit keeps only a
// few warps busy (its blocks form one chain): the number of chains in flight
// is what the device's throughput follows, and with gangs it is not limited
// by the number of hardware queues.
constexpr int kMaxGang = 32;
constexpr int kCallLanes = 16;  // lanes (host threads) a call spreads over (measured: 8, 16
                                // and 32 lanes give the same throughput; fewer lanes = fewer
                                // host threads and fewer launches)

int
code_raht(bool forward, const pccb200_raht_params& pp, const std::vector<RahtUnit>& given)
{
  std::vector<RahtUnit> units;
  for (const RahtUnit& u : given) {
    bool fuse = u.numSets > 1 && u.n >= 2 && !u.qpo;  // (same test as raht_run_sets)
    for (int s = 0; s < u.numSets && fuse; s++)
      fuse = WaveDescent<DeviceExec>::enabled(make_config(pp, *u.qs[s], forward, u.A[s], false));
    if (fuse || u.numSets == 1)
      units.push_back(u);
    else
      for (int s = 0; s < u.numSets; s++)
        units.push_back(u.only(s));
  }
  const int numUnits = int(units.size());
  // units per gang: by default the units are spread over all lanes first
  // (PCCB200_GANG: A/B knob, read per call)
  const char* eg = getenv("PCCB200_GANG");
  const int envGang = eg ? atoi(eg) : 0;
  int gang = envGang > 0 ? envGang : (numUnits + kCallLanes - 1) / kCallLanes;
  gang = gang > kMaxGang ? kMaxGang : gang;
  const int numGangs = (numUnits + gang - 1) / gang;
  return parallel_for(numGangs, kMaxLanes, [&](int g) -> int {
    const int u0 = g * gang;
    const int m = u0 + gang < numUnits ? gang : numUnits - u0;
    return with_device([&](DeviceExec& ex) -> int {
      return code_units(ex, forward, pp, units.data() + u0, m);
    });
  });
}

// one attribute, one unit per slice (coefficients: [A, total] planes)
int
attr_raht_slices(bool forward, bool dev, const pccb200_raht_params* params,
                 const pccb200_qpset* qpset, const int32_t* qpo, const int32_t* xyz,
                 int32_t* attrs, int A, int bitdepth, const int64_t* sliceOffsets, int numSlices,
                 int32_t* coeffs)
{
  int rc = check_slices(params, qpset, xyz, attrs, coeffs, A, bitdepth, sliceOffsets, numSlices);
  if (rc != PCCB200_OK)
    return rc;
  std::vector<RahtUnit> units(numSlices);
  for (int s = 0; s < numSlices; s++) {
    const int64_t o = sliceOffsets[s];
    RahtUnit& u = units[s];
    u.n = int(sliceOffsets[s + 1] - o);
    u.xyz = xyz + 3 * o;
    u.qpo = qpo ? qpo + 2 * o : nullptr;
    u.dev = dev;
    u.numSets = 1;
    u.qs[0] = qpset;
    u.A[0] = A;
    u.bitdepth[0] = bitdepth;
    u.attrs[0] = attrs + o * A;
    u.coef[0] = coeffs + o;
    u.coefStride[0] = sliceOffsets[numSlices];
  }
  return code_raht(forward, *params, units);
}

// several attributes of one unit per xyz[u] (coefficients: [A_s, n[u]] planes);
// attrs / coeffs hold numSets pointers per unit
int
attr_raht_units(bool forward, bool dev, const pccb200_raht_params* params, int numSets,
                const pccb200_qpset* const* qpsets, int numUnits, const int32_t* const* xyz,
                int32_t* const* attrs, const int32_t* A, const int32_t* bitdepth,
                const int32_t* n, int32_t* const* coeffs)
{
  std::vector<RahtUnit> units(numUnits);
  for (int i = 0; i < numUnits; i++) {
    RahtUnit& u = units[i];
    u.n = n[i];
    u.xyz = xyz[i];
    u.dev = dev;
    u.numSets = numSets;
    for (int s = 0; s < numSets; s++) {
      u.qs[s] = qpsets[s];
      u.A[s] = A[s];
      u.bitdepth[s] = bitdepth[s];
      u.attrs[s] = attrs[size_t(i) * numSets + s];
      u.coef[s] = coeffs[size_t(i) * numSets + s];
      u.coefStride[s] = n[i];
    }
  }
  return code_raht(forward, *params, units);
}

int
attr_raht_multi(bool forward, bool dev, const pccb200_raht_params* params, int numSets,
                const pccb200_qpset* const* qpsets, const int32_t* xyz, int32_t* const* attrs,
                const int32_t* A, const int32_t* bitdepth, int32_t n, int32_t* const* coeffs)
{
  int rc = check_multi(params, numSets, qpsets, xyz, reinterpret_cast<const void* const*>(attrs),
                       A, bitdepth, reinterpret_cast<const void* const*>(coeffs), n);
  if (rc != PCCB200_OK)
    return rc;
  return attr_raht_units(forward, dev, params, numSets, qpsets, 1, &xyz, attrs, A, bitdepth, &n,
                         coeffs);
}

int
attr_raht_batch(bool forward, bool dev, const pccb200_raht_params* params, int numSets,
                const pccb200_qpset* const* qpsets, int numUnits, const int32_t* const* xyz,
                int32_t* const* attrs, const int32_t* A, const int32_t* bitdepth,
                const int32_t* n, int32_t* const* coeffs)
{
  if (!xyz || !attrs || !coeffs || !n || numUnits <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  for (int u = 0; u < numUnits; u++) {
    if (!xyz[u])
      return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
    int rc = check_multi(params, numSets, qpsets, xyz[u],
                         reinterpret_cast<const void* const*>(attrs + size_t(u) * numSets), A,
                         bitdepth, reinterpret_cast<const void* const*>(coeffs + size_t(u) * numSets),
                         n[u]);
    if (rc != PCCB200_OK)
      return rc;
  }
  return attr_raht_units(forward, dev, params, numSets, qpsets, numUnits, xyz, attrs, A, bitdepth,
                         n, coeffs);
}

// One coding unit of an attribute-lifting call (a slice, or a whole frame): n
// points, optional point qp offsets ([n, 2]), its levels of detail (lod's, or
// the handle's) and 1..kLiftMaxSets attribute sets.  Per set: attrsIn ==
// attrsOut ([n, A], in and out), values ([n, A], coding order) and lcp, the
// caller's row of PCCB200_MAX_LODS LCP coefficients (or null).  dev: device
// pointers, attrs coded in place; otherwise host pointers.
struct LiftUnit {
  int n = 0;
  const int32_t* xyz = nullptr;
  const int32_t* qpo = nullptr;
  bool dev = false;
  const pccb200_lod_params* lod = nullptr;
  const pccb200_lod_scalable* scal = nullptr;  // scalable lifting, or null
  pccb200_lod_handle handle = nullptr;
  int numSets = 0;
  LiftSet sets[kLiftMaxSets] = {};
};

// Validated units over at most kCallLanes lanes, one lane each: stage in, build
// the levels of detail (or take the handle's), attr_lift_on_lods, stage out.
// nameUnits: a failure's message names the unit.
int
code_lift(bool forward, const std::vector<LiftUnit>& units, bool nameUnits)
{
  return parallel_for(int(units.size()), kCallLanes, [&](int i) -> int {
    const LiftUnit& u = units[i];
    const std::string unit = nameUnits ? "unit " + std::to_string(i) + ": " : std::string();
    pccb200_lod_handle h = u.handle;
    if (h && h->device != ctx().device)
      return fail(PCCB200_ERR_INVALID_ARG, unit + "handle belongs to another device");
    const int levels = u.scal ? kScalableLevels : u.lod->num_detail_levels;
    int8_t lcpLocal[kLiftMaxSets][PCCB200_MAX_LODS + 1] = {};
    for (int s = 0; s < u.numSets; s++)
      if (!forward && u.sets[s].lcpEnabled && u.sets[s].A == 3)
        for (int l = 0; l < levels && l < PCCB200_MAX_LODS; l++)
          lcpLocal[s][l] = u.sets[s].lcp[l];
    int rc = with_device([&](DeviceExec& ex) -> int {
      const int32_t* dXyz = u.dev || !u.xyz ? u.xyz : to_device(ex, u.xyz, size_t(u.n) * 3);
      const int32_t* dQpo = u.dev || !u.qpo ? u.qpo : to_device(ex, u.qpo, size_t(u.n) * 2);
      LiftSet sets[kLiftMaxSets];
      for (int s = 0; s < u.numSets; s++) {
        const LiftSet& t = u.sets[s];
        const size_t len = size_t(u.n) * t.A;
        sets[s] = t;
        sets[s].lcp = lcpLocal[s];
        if (u.dev)
          continue;
        sets[s].attrsIn = forward ? to_device(ex, t.attrsIn, len) : nullptr;
        sets[s].values = forward ? ex.alloc<int32_t>(len) : to_device(ex, t.values, len);
        // (in place: the gather reads attrs before the final write-back overwrites it)
        sets[s].attrsOut = ex.alloc<int32_t>(len);
      }
      if (h) {
        std::lock_guard<std::mutex> g(h->qwMu);
        if (!h->qwReady) {
          const uint64_t geomPoints = h->scal.geom_num_points ? h->scal.geom_num_points : u.n;
          int rcq = h->scalable
                      ? run_quant_weights_scalable(ex, h->st.npl, h->st.lodCount, geomPoints,
                                                   h->scal.min_geom_node_size_log2, u.n, h->st.qw)
                      : run_quant_weights(ex, h->st.preds, u.n, h->st.npl, h->st.lodCount,
                                          h->st.qw);
          if (rcq != PCCB200_OK)
            return fail(rcq, unit + "invalid levels of detail");
          PCC_CUDA_CHECK(cudaStreamSynchronize(ex.stream));  // other lanes read them from now on
          h->qwReady = true;
        }
      }
      int rc2 = h ? attr_lift_on_lods(ex, forward, h->st, dQpo, u.numSets, sets)
                  : attr_lift_run(ex, forward, *u.lod, dQpo, dXyz, u.n, u.numSets, sets, u.scal);
      if (rc2 != PCCB200_OK)
        return fail(rc2, unit + (rc2 == PCCB200_ERR_UNSUPPORTED
                                   ? "a predictor references its own level of detail"
                                   : "invalid lifting parameters"));
      for (int s = 0; s < u.numSets && !u.dev; s++) {
        const size_t len = size_t(u.n) * u.sets[s].A;
        to_host(ex, u.sets[s].attrsOut, sets[s].attrsOut, len);
        if (forward)
          to_host(ex, u.sets[s].values, sets[s].values, len);
      }
      return PCCB200_OK;
    });
    for (int s = 0; s < u.numSets && rc == PCCB200_OK && forward; s++)
      if (u.sets[s].lcp)
        for (int l = 0; l < levels && l < PCCB200_MAX_LODS; l++)
          u.sets[s].lcp[l] = lcpLocal[s][l];
    return rc;
  });
}

// Slices of a frame (tmc3/encoder.cpp:545-568), each with its own levels of
// detail: slice s is points [offs[s], offs[s + 1]) and row s of lcp.  With a
// handle h: the one slice it was made for (lod, xyz and offs are not read).
int
attr_lift(bool forward, bool dev, const pccb200_lod_params* lod, pccb200_lod_handle h,
          const pccb200_qpset* qpset, int32_t lcpEnabled, const int32_t* qpo, const int32_t* xyz,
          int32_t* attrs, int32_t A, int32_t bitdepth, const int64_t* offs, int32_t numSlices,
          int32_t* values, int8_t* lcp)
{
  const int64_t whole[2] = {0, h ? h->st.n : 0};
  if (h) {
    lod = &h->params;
    offs = whole;
    numSlices = 1;
  }
  int rc = check_offsets(offs, numSlices);
  if (rc != PCCB200_OK)
    return rc;
  if (!lod || (!h && !xyz) || !qpset || !attrs || !values || (A != 1 && A != 3) || bitdepth < 1
      || bitdepth > 16)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  if (!forward && lcpEnabled && A == 3 && !lcp)
    return fail(PCCB200_ERR_INVALID_ARG, "lcp coefficients missing");
  std::vector<LiftUnit> units(numSlices);
  for (int s = 0; s < numSlices; s++) {
    const int64_t o = offs[s];
    LiftUnit& u = units[s];
    u.n = int(offs[s + 1] - o);
    u.xyz = h ? nullptr : xyz + 3 * o;
    u.qpo = qpo ? qpo + 2 * o : nullptr;
    u.dev = dev;
    u.lod = lod;
    u.handle = h;
    u.numSets = 1;
    u.sets[0] = LiftSet{A, bitdepth, qpset, lcpEnabled != 0, attrs + o * A, attrs + o * A,
                        values + o * A, lcp ? lcp + size_t(s) * PCCB200_MAX_LODS : nullptr};
  }
  return code_lift(forward, units, false);
}

// Checks the arguments of a pccb200_attr_lift_*_multi* call, before any device
// is looked up, and describes its units.  Unit u: lods[u], xyz[u], n[u], and
// per set s attrs / values / lcp[u * numSets + s]; qpsets, lcpEnabled, A and
// bitdepth are per set.  lcp (the whole array) may be null when no set needs it.
int
lift_units(bool forward, bool dev, int numUnits, const pccb200_lod_params* const* lods,
           int numSets, const pccb200_qpset* const* qpsets, const int32_t* lcpEnabled,
           const int32_t* const* xyz, const int32_t* n, int32_t* const* attrs, const int32_t* A,
           const int32_t* bitdepth, int32_t* const* values, int8_t* const* lcp,
           std::vector<LiftUnit>& units)
{
  if (!lods || !qpsets || !lcpEnabled || !xyz || !n || !attrs || !A || !bitdepth || !values
      || numUnits <= 0 || numSets < 1 || numSets > kLiftMaxSets)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  for (int s = 0; s < numSets; s++)
    if (!qpsets[s] || (A[s] != 1 && A[s] != 3) || bitdepth[s] < 1 || bitdepth[s] > 16)
      return fail(PCCB200_ERR_INVALID_ARG,
                  "set " + std::to_string(s) + ": null qpset, bad component count or bit depth");
  units.resize(numUnits);
  for (int i = 0; i < numUnits; i++) {
    const std::string unit = "unit " + std::to_string(i) + ": ";
    LiftUnit& u = units[i];
    u.n = n[i];
    u.xyz = xyz[i];
    u.dev = dev;
    u.lod = lods[i];
    u.numSets = numSets;
    if (!u.lod || !u.xyz)
      return fail(PCCB200_ERR_INVALID_ARG, unit + "null pointer");
    if (u.n <= 0)
      return fail(PCCB200_ERR_INVALID_ARG, unit + "no points");
    for (int s = 0; s < numSets; s++) {
      const size_t at = size_t(i) * numSets + s;
      int8_t* row = lcp ? lcp[at] : nullptr;
      if (!attrs[at] || !values[at])
        return fail(PCCB200_ERR_INVALID_ARG, unit + "null pointer");
      if (!forward && lcpEnabled[s] && A[s] == 3 && !row)
        return fail(PCCB200_ERR_INVALID_ARG, unit + "lcp coefficients missing");
      u.sets[s] = LiftSet{A[s], bitdepth[s], qpsets[s], lcpEnabled[s] != 0, attrs[at], attrs[at],
                          values[at], row};
    }
  }
  return PCCB200_OK;
}

// The scalable-lifting arguments a host can check: the encoder codes whole
// slices (the reference calls AttributeLods::generate with minGeomNodeSizeLog2
// = 0 and computeQuantizationWeightsScalable with (n, 0)).
int
check_scalable(const pccb200_lod_params& lod, const pccb200_lod_scalable& sc, int n, bool encoder,
               const std::string& unit)
{
  if (lod.lod_decimation_type != 0)
    return fail(PCCB200_ERR_INVALID_ARG, unit + "scalable lifting needs lod_decimation_type 0");
  if (sc.max_neigh_range < 1 || sc.reserved != 0)
    return fail(PCCB200_ERR_INVALID_ARG, unit + "max_neigh_range < 1 or reserved not 0");
  if (sc.min_geom_node_size_log2 < 0 || sc.min_geom_node_size_log2 >= kScalableLevels
      || (sc.geom_num_points != 0 && sc.geom_num_points < n))
    return fail(PCCB200_ERR_INVALID_ARG,
                unit + "min_geom_node_size_log2 out of range or geom_num_points < n");
  if (encoder && (sc.min_geom_node_size_log2 != 0 || (sc.geom_num_points != 0
                                                       && sc.geom_num_points != n)))
    return fail(PCCB200_ERR_INVALID_ARG, unit + "the encoder codes whole slices");
  return PCCB200_OK;
}

int
attr_lift_scalable(bool forward, bool dev, int numUnits, const pccb200_lod_params* const* lods,
                   const pccb200_lod_scalable* scals, int numSets,
                   const pccb200_qpset* const* qpsets, const int32_t* lcpEnabled,
                   const int32_t* const* xyz, const int32_t* n, int32_t* const* attrs,
                   const int32_t* A, const int32_t* bitdepth, int32_t* const* values,
                   int8_t* const* lcp)
{
  if (!scals)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  std::vector<LiftUnit> units;
  int rc = lift_units(forward, dev, numUnits, lods, numSets, qpsets, lcpEnabled, xyz, n, attrs, A,
                      bitdepth, values, lcp, units);
  if (rc != PCCB200_OK)
    return rc;
  for (int i = 0; i < numUnits; i++) {
    rc = check_scalable(*lods[i], scals[i], n[i], forward, "unit " + std::to_string(i) + ": ");
    if (rc != PCCB200_OK)
      return rc;
    units[i].scal = &scals[i];
  }
  return code_lift(forward, units, true);
}

int
attr_lift_multi(bool forward, bool dev, int numUnits, const pccb200_lod_params* const* lods,
                int numSets, const pccb200_qpset* const* qpsets, const int32_t* lcpEnabled,
                const int32_t* const* xyz, const int32_t* n, int32_t* const* attrs,
                const int32_t* A, const int32_t* bitdepth, int32_t* const* values,
                int8_t* const* lcp)
{
  std::vector<LiftUnit> units;
  int rc = lift_units(forward, dev, numUnits, lods, numSets, qpsets, lcpEnabled, xyz, n, attrs, A,
                      bitdepth, values, lcp, units);
  if (rc != PCCB200_OK)
    return rc;
  return code_lift(forward, units, true);
}

// One unit of a recolouring call (a slice, or a whole frame): source and
// target positions, scale and offset, and per attribute set its source values,
// component count, bit depth and output (sets[s].refined1 is not used here).
// dev: device pointers; otherwise host pointers.
struct RecolourUnit {
  int nSrc = 0, nTgt = 0;
  const int32_t* srcXyz = nullptr;
  const int32_t* tgtXyz = nullptr;
  double scale = 1.0;
  int32_t off[3] = {};
  bool dev = false;
  int numSets = 0;
  RecolourSet sets[kRecolourMaxSets] = {};
  RecolourSearch search = kRecolourGrid;
};

// Validated units over at most kCallLanes lanes, one lane each: stage in,
// recolour_run, stage out.  nameUnits: a failure's message names the unit.
int
code_recolour(const pccb200_recolour_params& rp, const std::vector<RecolourUnit>& units,
              bool nameUnits)
{
  return parallel_for(int(units.size()), kCallLanes, [&](int i) -> int {
    const RecolourUnit& u = units[i];
    return with_device([&](DeviceExec& ex) -> int {
      RecolourSet sets[kRecolourMaxSets];
      const int32_t* dSrc = u.dev ? u.srcXyz : to_device(ex, u.srcXyz, size_t(u.nSrc) * 3);
      for (int s = 0; s < u.numSets; s++) {
        sets[s] = u.sets[s];
        if (!u.dev)
          sets[s].srcAttr = to_device(ex, u.sets[s].srcAttr, size_t(u.nSrc) * u.sets[s].A);
      }
      const int32_t* dTgt = u.dev ? u.tgtXyz : to_device(ex, u.tgtXyz, size_t(u.nTgt) * 3);
      for (int s = 0; s < u.numSets && !u.dev; s++)
        sets[s].out = ex.alloc<int32_t>(size_t(u.nTgt) * u.sets[s].A);
      int rc = recolour_run(ex, rp, dSrc, u.nSrc, u.scale, u.off, dTgt, u.nTgt, u.numSets, sets,
                            u.search);
      if (rc != PCCB200_OK)
        return fail(rc, (nameUnits ? "unit " + std::to_string(i) + ": " : std::string())
                          + (u.search == kRecolourRefExact
                               ? "invalid recolouring parameters (neighbour counts, scale, or a "
                                 "coordinate or offset outside (-2^30, 2^30))"
                               : "invalid recolouring parameters (neighbour counts, scale, or a "
                                 "coordinate outside [0, 2^21))"));
      for (int s = 0; s < u.numSets && !u.dev; s++)
        to_host(ex, u.sets[s].out, sets[s].out, size_t(u.nTgt) * u.sets[s].A);
      return PCCB200_OK;
    });
  });
}

// Checks the arguments of a pccb200_recolour_multi* call, before any device is
// looked up, and describes its units.  Unit u: srcXyz[u], tgtXyz[u], scale[u],
// offsets[3u..3u+2], and per set s srcAttrs[u * numSets + s], out[u * numSets + s].
int
recolour_units(bool dev, const pccb200_recolour_params* params, int numSets, int numUnits,
               const int32_t* const* srcXyz, const int32_t* nSrc,
               const int32_t* const* srcAttrs, const int32_t* A, const int32_t* bitdepth,
               const double* scale, const int32_t* offsets, const int32_t* const* tgtXyz,
               const int32_t* nTgt, int32_t* const* out, std::vector<RecolourUnit>& units,
               RecolourSearch search)
{
  if (!params || !srcXyz || !nSrc || !srcAttrs || !A || !bitdepth || !scale || !offsets
      || !tgtXyz || !nTgt || !out || numUnits <= 0 || numSets < 1 || numSets > kRecolourMaxSets)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  units.resize(numUnits);
  for (int i = 0; i < numUnits; i++) {
    RecolourUnit& u = units[i];
    u.nSrc = nSrc[i];
    u.nTgt = nTgt[i];
    u.srcXyz = srcXyz[i];
    u.tgtXyz = tgtXyz[i];
    u.scale = scale[i];
    for (int k = 0; k < 3; k++)
      u.off[k] = offsets[3 * size_t(i) + k];
    u.dev = dev;
    u.numSets = numSets;
    u.search = search;
    bool null = !u.srcXyz || !u.tgtXyz;
    for (int s = 0; s < numSets; s++) {
      const size_t at = size_t(i) * numSets + s;
      u.sets[s] = RecolourSet{srcAttrs[at], A[s], bitdepth[s], nullptr, out[at]};
      null = null || !srcAttrs[at] || !out[at];
    }
    if (null)
      return fail(PCCB200_ERR_INVALID_ARG, "unit " + std::to_string(i) + ": null pointer");
    if (!recolour_args_valid(*params, u.nSrc, u.nTgt, u.scale, numSets, u.sets))
      return fail(PCCB200_ERR_INVALID_ARG,
                  "unit " + std::to_string(i) + ": bad point count, neighbour count, component "
                  "count, bit depth, search range or scale");
  }
  return PCCB200_OK;
}

int
recolour_multi(bool dev, const pccb200_recolour_params* params, int numSets, int numUnits,
               const int32_t* const* srcXyz, const int32_t* nSrc,
               const int32_t* const* srcAttrs, const int32_t* A, const int32_t* bitdepth,
               const double* scale, const int32_t* offsets, const int32_t* const* tgtXyz,
               const int32_t* nTgt, int32_t* const* out, RecolourSearch search = kRecolourGrid)
{
  std::vector<RecolourUnit> units;
  int rc = recolour_units(dev, params, numSets, numUnits, srcXyz, nSrc, srcAttrs, A, bitdepth,
                          scale, offsets, tgtXyz, nTgt, out, units, search);
  if (rc != PCCB200_OK)
    return rc;
  return code_recolour(*params, units, true);
}

// One unit of a predicting-transform decode: the handle's levels of detail, or
// lod and xyz; qp offsets ([n, 2]) or null; per set the caller's values_in and
// attrs_out ([n, A]) and ICP row.  dev: device pointers, otherwise host ones.
struct PredCallUnit {
  int n = 0;
  const int32_t* xyz = nullptr;
  const int32_t* qpo = nullptr;
  const pccb200_lod_params* lod = nullptr;
  pccb200_lod_handle handle = nullptr;
  PredUnit pu = {};
};

// Validated units dealt over at most kCallLanes lanes (unit u to lane
// u % lanes); the units of a lane form one gang: levels of detail, then one
// attr_pred_decode_on_lods (one dataflow launch) for all of them.
int
code_pred(bool dev, const std::vector<PredCallUnit>& units)
{
  const int numUnits = int(units.size());
  const int lanes = numUnits < kCallLanes ? numUnits : kCallLanes;
  return parallel_for(lanes, lanes, [&](int g) -> int {
    std::vector<int> mine;
    for (int u = g; u < numUnits; u += lanes)
      mine.push_back(u);
    for (int u : mine)
      if (units[u].handle && units[u].handle->device != ctx().device)
        return fail(PCCB200_ERR_INVALID_ARG, "unit " + std::to_string(u)
                                               + ": handle belongs to another device");
    return with_device([&](DeviceExec& ex) -> int {
      std::vector<LodState> st(mine.size());
      std::vector<PredUnit> pu(mine.size());
      for (size_t m = 0; m < mine.size(); m++) {
        const PredCallUnit& cu = units[mine[m]];
        const std::string unit = "unit " + std::to_string(mine[m]) + ": ";
        const size_t n = size_t(cu.n);
        if (cu.handle) {
          st[m] = cu.handle->st;
        } else {
          st[m].preds = ex.alloc<pccb200_predictor>(n);
          st[m].idx = ex.alloc<uint32_t>(n);
          st[m].qw = nullptr;
          const int32_t* dXyz = dev ? cu.xyz : to_device(ex, cu.xyz, n * 3);
          int rc = lod_state_build(ex, *cu.lod, dXyz, cu.n, st[m], false);
          if (rc != PCCB200_OK)
            return fail(rc, unit + "invalid LoD parameters");
        }
        pu[m] = cu.pu;
        pu[m].st = &st[m];
        pu[m].qpo = dev || !cu.qpo ? cu.qpo : to_device(ex, cu.qpo, n * 2);
        for (int s = 0; s < pu[m].numSets && !dev; s++) {
          const size_t len = n * pu[m].sets[s].A;
          pu[m].sets[s].values = to_device(ex, cu.pu.sets[s].values, len);
          pu[m].sets[s].attrsOut = ex.alloc<int32_t>(len);
        }
      }
      int bad = 0;
      const char* why = "invalid predicting-transform parameters";
      int rc = attr_pred_decode_on_lods(ex, int(mine.size()), pu.data(), &bad, &why);
      if (rc != PCCB200_OK)
        return fail(rc, "unit " + std::to_string(mine[bad]) + ": " + why);
      for (size_t m = 0; m < mine.size() && !dev; m++)
        for (int s = 0; s < pu[m].numSets; s++)
          to_host(ex, units[mine[m]].pu.sets[s].attrsOut, pu[m].sets[s].attrsOut,
                  size_t(units[mine[m]].n) * pu[m].sets[s].A);
      return PCCB200_OK;
    });
  });
}

int
check_pred_set(const pccb200_qpset* qs, const pccb200_pred_params* pp, int A, int bitdepth)
{
  if (!qs || !pp || (A != 1 && A != 3) || bitdepth < 1 || bitdepth > 16)
    return PCCB200_ERR_INVALID_ARG;
  if (qs->num_layers < 1 || qs->num_layers > PCCB200_MAX_QP_LAYERS)
    return PCCB200_ERR_INVALID_ARG;
  if (pp->max_num_direct_predictors < 0 || pp->max_num_direct_predictors > 3
      || pp->adaptive_prediction_threshold < 0 || pp->adaptive_prediction_threshold > 255)
    return PCCB200_ERR_INVALID_ARG;
  return PCCB200_OK;
}

int
attr_pred_multi(bool dev, int numUnits, const pccb200_lod_params* const* lods,
                const int32_t* qnw, int numSets, const pccb200_qpset* const* qpsets,
                const pccb200_pred_params* pred, const int32_t* A, const int32_t* bitdepth,
                const int32_t* const* xyz, const int32_t* n, const int32_t* const* qpo,
                const int32_t* const* values, const int8_t* const* icp, int32_t* const* out)
{
  if (!lods || !qnw || !qpsets || !pred || !A || !bitdepth || !xyz || !n || !values || !out
      || numUnits <= 0 || numSets < 1 || numSets > kPredMaxSets)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  for (int s = 0; s < numSets; s++)
    if (check_pred_set(qpsets[s], &pred[s], A[s], bitdepth[s]) != PCCB200_OK)
      return fail(PCCB200_ERR_INVALID_ARG,
                  "set " + std::to_string(s)
                    + ": null pointer, bad component count, bit depth, qp layers or "
                      "predicting-transform parameters");
  std::vector<PredCallUnit> units(numUnits);
  for (int u = 0; u < numUnits; u++) {
    const std::string unit = "unit " + std::to_string(u) + ": ";
    PredCallUnit& cu = units[u];
    cu.n = n[u];
    cu.xyz = xyz[u];
    cu.qpo = qpo ? qpo[u] : nullptr;
    cu.lod = lods[u];
    if (!cu.lod || !cu.xyz)
      return fail(PCCB200_ERR_INVALID_ARG, unit + "null pointer");
    if (cu.n <= 0)
      return fail(PCCB200_ERR_INVALID_ARG, unit + "no points");
    for (int k = 0; k < 3; k++)
      cu.pu.quantNeighWeight[k] = qnw[3 * u + k];
    cu.pu.numSets = numSets;
    for (int s = 0; s < numSets; s++) {
      const size_t at = size_t(u) * numSets + s;
      if (!values[at] || !out[at])
        return fail(PCCB200_ERR_INVALID_ARG, unit + "null pointer");
      cu.pu.sets[s] = PredSet{A[s], bitdepth[s], qpsets[s], pred[s], values[at],
                              icp ? icp[at] : nullptr, out[at]};
    }
  }
  return code_pred(dev, units);
}

}  // namespace
}  // namespace pccb200

using namespace pccb200;

extern "C" {

void
pccb200_raht_set_prediction_weights(pccb200_raht_params* p, const int32_t w[5])
{
  const int child[12] = {4, 4, 3, 4, 3, 3, 4, 4, 4, 4, 4, 4};
  const int parent[19] = {0, 1, 1, 1, 2, 2, 2, 2, 2, 1, 2, 1, 1, 2, 2, 2, 2, 2, 2};
  for (int i = 0; i < 12; i++)
    p->pred_weight_child[i] = w[child[i]];
  for (int i = 0; i < 19; i++)
    p->pred_weight_parent[i] = w[parent[i]];
}

void
pccb200_raht_params_default(pccb200_raht_params* p)
{
  p->prediction_enabled = 1;
  p->integer_haar = 0;
  p->prediction_threshold0 = 2;
  p->prediction_threshold1 = 6;
  p->subnode_prediction_enabled = 1;
  p->prediction_search_range = 50000;
  p->raht_extension = 1;
  const int32_t w[5] = {9, 3, 1, 5, 2};
  pccb200_raht_set_prediction_weights(p, w);
}

int
pccb200_abi_version(void)
{
  return PCCB200_ABI_VERSION;
}

int
pccb200_set_device(int device)
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  if (device < 0)
    return fail(PCCB200_ERR_INVALID_ARG, "negative device index");
  if (c.ready && device != c.device) {
    if (c.active.load())
      return fail(PCCB200_ERR_INVALID_ARG, "calls in flight on the current device");
    cudaSetDevice(c.device);
    destroy_lanes(c);
    if (c.timeStream) {
      cudaEventDestroy(c.timeBegin);
      cudaEventDestroy(c.timeEnd);
      cudaStreamDestroy(c.timeStream);
      c.timeStream = nullptr;
    }
    c.ready = false;
  }
  c.device = device;
  return ensure_ready(c);
}

const char*
pccb200_last_error(void)
{
  return t_lastError.c_str();
}

uint64_t
pccb200_kernel_launch_count(void)
{
  return g_launchCount.load();
}

int
pccb200_morton_sort(const int32_t* xyz, int32_t n, int64_t* keys_out, int32_t* order_out)
{
  if (!xyz || !keys_out || !order_out || n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    int64_t* dKeys = ex.alloc<int64_t>(n);
    int32_t* dOrder = ex.alloc<int32_t>(n);
    device_morton_sort(ex, dXyz, n, dKeys, dOrder);
    to_host(ex, keys_out, dKeys, size_t(n));
    to_host(ex, order_out, dOrder, size_t(n));
    return PCCB200_OK;
  });
}

int
pccb200_raht_forward(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                     const int32_t* point_qp_offsets, const int64_t* morton,
                     int32_t* attrs_inout, int32_t num_attrs, int32_t n,
                     int32_t* coeffs_out)
{
  return raht_common(true, params, qpset, point_qp_offsets, morton, attrs_inout, num_attrs, n,
                     coeffs_out);
}

int
pccb200_raht_inverse(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                     const int32_t* point_qp_offsets, const int64_t* morton,
                     int32_t* attrs_out, int32_t num_attrs, int32_t n,
                     const int32_t* coeffs_in)
{
  return raht_common(false, params, qpset, point_qp_offsets, morton, attrs_out, num_attrs, n,
                     const_cast<int32_t*>(coeffs_in));
}

int
pccb200_attr_raht_encode(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                         const int32_t* point_qp_offsets, const int32_t* xyz,
                         int32_t* attrs_inout, int32_t num_attrs, int32_t n, int32_t bitdepth,
                         int32_t* coeffs_out)
{
  const int64_t offs[2] = {0, n};
  return attr_raht_slices(true, false, params, qpset, point_qp_offsets, xyz, attrs_inout, num_attrs,
                          bitdepth, offs, 1, coeffs_out);
}

int
pccb200_attr_raht_decode(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                         const int32_t* point_qp_offsets, const int32_t* xyz,
                         int32_t* attrs_out, int32_t num_attrs, int32_t n, int32_t bitdepth,
                         const int32_t* coeffs_in)
{
  const int64_t offs[2] = {0, n};
  return attr_raht_slices(false, false, params, qpset, point_qp_offsets, xyz, attrs_out, num_attrs,
                          bitdepth, offs, 1, const_cast<int32_t*>(coeffs_in));
}

int
pccb200_attr_raht_encode_slices(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                                const int32_t* point_qp_offsets, const int32_t* xyz,
                                int32_t* attrs_inout, int32_t num_attrs, int32_t bitdepth,
                                const int64_t* slice_offsets, int32_t num_slices,
                                int32_t* coeffs_out)
{
  return attr_raht_slices(true, false, params, qpset, point_qp_offsets, xyz, attrs_inout, num_attrs,
                          bitdepth, slice_offsets, num_slices, coeffs_out);
}

int
pccb200_attr_raht_encode_slices_dev(const pccb200_raht_params* params,
                                    const pccb200_qpset* qpset,
                                    const int32_t* d_point_qp_offsets, const int32_t* d_xyz,
                                    int32_t* d_attrs_inout, int32_t num_attrs, int32_t bitdepth,
                                    const int64_t* slice_offsets, int32_t num_slices,
                                    int32_t* d_coeffs_out)
{
  return attr_raht_slices(true, true, params, qpset, d_point_qp_offsets, d_xyz, d_attrs_inout,
                          num_attrs, bitdepth, slice_offsets, num_slices, d_coeffs_out);
}

int
pccb200_attr_raht_decode_slices_dev(const pccb200_raht_params* params,
                                    const pccb200_qpset* qpset,
                                    const int32_t* d_point_qp_offsets, const int32_t* d_xyz,
                                    int32_t* d_attrs_out, int32_t num_attrs, int32_t bitdepth,
                                    const int64_t* slice_offsets, int32_t num_slices,
                                    const int32_t* d_coeffs_in)
{
  return attr_raht_slices(false, true, params, qpset, d_point_qp_offsets, d_xyz, d_attrs_out,
                          num_attrs, bitdepth, slice_offsets, num_slices,
                          const_cast<int32_t*>(d_coeffs_in));
}

int
pccb200_attr_raht_encode_multi(const pccb200_raht_params* params, int32_t num_sets,
                               const pccb200_qpset* const* qpsets, const int32_t* xyz,
                               int32_t* const* attrs_inout, const int32_t* num_attrs,
                               const int32_t* bitdepths, int32_t n, int32_t* const* coeffs_out)
{
  return attr_raht_multi(true, false, params, num_sets, qpsets, xyz, attrs_inout,
                         num_attrs, bitdepths, n, coeffs_out);
}

int
pccb200_attr_raht_decode_multi(const pccb200_raht_params* params, int32_t num_sets,
                               const pccb200_qpset* const* qpsets, const int32_t* xyz,
                               int32_t* const* attrs_out, const int32_t* num_attrs,
                               const int32_t* bitdepths, int32_t n,
                               const int32_t* const* coeffs_in)
{
  return attr_raht_multi(false, false, params, num_sets, qpsets, xyz, attrs_out,
                         num_attrs, bitdepths, n,
                         const_cast<int32_t* const*>(coeffs_in));
}

int
pccb200_attr_raht_encode_multi_dev(const pccb200_raht_params* params, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* d_xyz,
                                   int32_t* const* d_attrs_inout, const int32_t* num_attrs,
                                   const int32_t* bitdepths, int32_t n,
                                   int32_t* const* d_coeffs_out)
{
  return attr_raht_multi(true, true, params, num_sets, qpsets, d_xyz, d_attrs_inout,
                         num_attrs, bitdepths, n, d_coeffs_out);
}

int
pccb200_attr_raht_decode_multi_dev(const pccb200_raht_params* params, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* d_xyz,
                                   int32_t* const* d_attrs_out, const int32_t* num_attrs,
                                   const int32_t* bitdepths, int32_t n,
                                   const int32_t* const* d_coeffs_in)
{
  return attr_raht_multi(false, true, params, num_sets, qpsets, d_xyz, d_attrs_out,
                         num_attrs, bitdepths, n,
                         const_cast<int32_t* const*>(d_coeffs_in));
}

int
pccb200_attr_raht_encode_multi_batch(const pccb200_raht_params* params, int32_t num_sets,
                                     const pccb200_qpset* const* qpsets, int32_t num_units,
                                     const int32_t* const* xyz, int32_t* const* attrs_inout,
                                     const int32_t* num_attrs, const int32_t* bitdepths,
                                     const int32_t* n, int32_t* const* coeffs_out)
{
  return attr_raht_batch(true, false, params, num_sets, qpsets, num_units, xyz,
                         attrs_inout, num_attrs, bitdepths, n, coeffs_out);
}

int
pccb200_attr_raht_decode_multi_batch(const pccb200_raht_params* params, int32_t num_sets,
                                     const pccb200_qpset* const* qpsets, int32_t num_units,
                                     const int32_t* const* xyz, int32_t* const* attrs_out,
                                     const int32_t* num_attrs, const int32_t* bitdepths,
                                     const int32_t* n, const int32_t* const* coeffs_in)
{
  return attr_raht_batch(false, false, params, num_sets, qpsets, num_units, xyz, attrs_out,
                         num_attrs, bitdepths, n, const_cast<int32_t* const*>(coeffs_in));
}

int
pccb200_attr_raht_encode_multi_batch_dev(const pccb200_raht_params* params, int32_t num_sets,
                                         const pccb200_qpset* const* qpsets, int32_t num_units,
                                         const int32_t* const* d_xyz,
                                         int32_t* const* d_attrs_inout, const int32_t* num_attrs,
                                         const int32_t* bitdepths, const int32_t* n,
                                         int32_t* const* d_coeffs_out)
{
  return attr_raht_batch(true, true, params, num_sets, qpsets, num_units, d_xyz,
                         d_attrs_inout, num_attrs, bitdepths, n, d_coeffs_out);
}

int
pccb200_attr_raht_decode_multi_batch_dev(const pccb200_raht_params* params, int32_t num_sets,
                                         const pccb200_qpset* const* qpsets, int32_t num_units,
                                         const int32_t* const* d_xyz, int32_t* const* d_attrs_out,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         const int32_t* n, const int32_t* const* d_coeffs_in)
{
  return attr_raht_batch(false, true, params, num_sets, qpsets, num_units, d_xyz,
                         d_attrs_out, num_attrs, bitdepths, n,
                         const_cast<int32_t* const*>(d_coeffs_in));
}


// Device-side timing across all lanes: begin() records an event that every
// lane's stream waits for; end() records one event that waits for every
// lane's stream and returns the elapsed milliseconds between the two.
int
pccb200_time_begin(void)
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  int rc = ensure_ready(c);
  if (rc != PCCB200_OK)
    return rc;
  cudaSetDevice(c.device);
  if (!c.timeStream) {
    cudaStreamCreateWithFlags(&c.timeStream, cudaStreamNonBlocking);
    cudaEventCreate(&c.timeBegin);
    cudaEventCreate(&c.timeEnd);
  }
  cudaEventRecord(c.timeBegin, c.timeStream);
  for (auto& l : c.lanes)
    cudaStreamWaitEvent(l->stream, c.timeBegin, 0);
  return PCCB200_OK;
}

int
pccb200_time_end(double* ms_out)
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  if (!c.timeStream || !ms_out)
    return fail(PCCB200_ERR_INVALID_ARG, "pccb200_time_begin not called");
  cudaSetDevice(c.device);
  for (auto& l : c.lanes) {
    cudaEventRecord(l->tail, l->stream);
    cudaStreamWaitEvent(c.timeStream, l->tail, 0);
  }
  cudaEventRecord(c.timeEnd, c.timeStream);
  cudaEventSynchronize(c.timeEnd);
  float ms = 0;
  if (cudaEventElapsedTime(&ms, c.timeBegin, c.timeEnd) != cudaSuccess)
    return fail(PCCB200_ERR_CUDA, "cudaEventElapsedTime failed");
  *ms_out = ms;
  return PCCB200_OK;
}

void
pccb200_profile_enable(int enable)
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  c.profEnabled = enable != 0;
}

void
pccb200_profile_reset(void)
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  for (int i = 0; i < PCCB200_NUM_PHASES; i++) {
    c.profMs[i] = 0;
    c.profLaunches[i] = 0;
  }
}

void
pccb200_profile_read(double ms_out[PCCB200_NUM_PHASES], uint64_t launches_out[PCCB200_NUM_PHASES])
{
  Context& c = ctx();
  std::lock_guard<std::mutex> lock(c.mu);
  for (int i = 0; i < PCCB200_NUM_PHASES; i++) {
    ms_out[i] = c.profMs[i];
    launches_out[i] = c.profLaunches[i];
  }
}

#ifdef PCCB200_HOP_STATS
// Developer build only (make hopstats; tools/hop_profile.py): the block
// kernel's cycle counters, kHopCounters values per descent step, read after a
// device synchronise and cleared.  Returns the number of values per step.
extern "C" int
pccb200_hop_stats_read(uint64_t* out, int32_t steps)
{
  static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "counter type");
  unsigned long long host[pccb200::kHopStages][pccb200::kHopCounters];
  if (cudaDeviceSynchronize() != cudaSuccess
      || cudaMemcpyFromSymbol(host, pccb200::g_hopStats, sizeof(host)) != cudaSuccess)
    return -1;
  for (int s = 0; s < steps && s < pccb200::kHopStages; s++)
    for (int c = 0; c < pccb200::kHopCounters; c++)
      out[size_t(s) * pccb200::kHopCounters + c] = host[s][c];
  memset(host, 0, sizeof(host));
  if (cudaMemcpyToSymbol(pccb200::g_hopStats, host, sizeof(host)) != cudaSuccess)
    return -1;
  return pccb200::kHopCounters;
}
#endif

int
pccb200_lod_build(const pccb200_lod_params* params, const int32_t* xyz, int32_t n,
                  pccb200_predictor* preds_out, uint32_t* indexes_out,
                  uint32_t* num_points_in_lod_out, int32_t* lod_count_out)
{
  if (!params || !xyz || !preds_out || !indexes_out || !num_points_in_lod_out || !lod_count_out
      || n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    pccb200_predictor* dP = ex.alloc<pccb200_predictor>(n);
    uint32_t* dIdx = ex.alloc<uint32_t>(n);
    int cnt = 0;
    int rc = lod_run(ex, *params, dXyz, n, dP, dIdx, num_points_in_lod_out, &cnt);
    if (rc != PCCB200_OK)
      return fail(rc, "invalid LoD parameters");
    *lod_count_out = cnt;
    to_host(ex, preds_out, dP, size_t(n));
    to_host(ex, indexes_out, dIdx, size_t(n));
    return PCCB200_OK;
  });
}

int
pccb200_lod_build_scalable(const pccb200_lod_params* params, const pccb200_lod_scalable* scal,
                           const int32_t* xyz, int32_t n, pccb200_predictor* preds_out,
                           uint32_t* indexes_out, uint32_t* num_points_in_lod_out,
                           int32_t* lod_count_out)
{
  if (!params || !scal || !xyz || !preds_out || !indexes_out || !num_points_in_lod_out
      || !lod_count_out || n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  int rc = check_scalable(*params, *scal, n, false, std::string());
  if (rc != PCCB200_OK)
    return rc;
  return with_device([&](DeviceExec& ex) -> int {
    int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    pccb200_predictor* dP = ex.alloc<pccb200_predictor>(n);
    uint32_t* dIdx = ex.alloc<uint32_t>(n);
    int cnt = 0;
    int rc2 = lod_run(ex, *params, dXyz, n, dP, dIdx, num_points_in_lod_out, &cnt, scal);
    if (rc2 != PCCB200_OK)
      return fail(rc2, "invalid LoD parameters");
    *lod_count_out = cnt;
    to_host(ex, preds_out, dP, size_t(n));
    to_host(ex, indexes_out, dIdx, size_t(n));
    return PCCB200_OK;
  });
}

// neighWeight: the fixed neighbour weights, or null for the distance-based ones
static int
quant_weights_common(const pccb200_predictor* preds, int32_t n, const uint32_t* num_points_in_lod,
                     int32_t lod_count, const int32_t* neighWeight, uint64_t* qw_out)
{
  if (!preds || !num_points_in_lod || !qw_out || n <= 0 || lod_count <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    pccb200_predictor* dP = to_device(ex, preds, size_t(n));
    uint64_t* dQw = ex.alloc<uint64_t>(n);
    int rc = run_quant_weights(ex, dP, n, num_points_in_lod, lod_count, dQw, neighWeight);
    if (rc != PCCB200_OK)
      return fail(rc, "numPointsInLod does not partition [0, n)");
    to_host(ex, qw_out, dQw, size_t(n));
    return PCCB200_OK;
  });
}

int
pccb200_quant_weights(const pccb200_predictor* preds, int32_t n,
                      const uint32_t* num_points_in_lod, int32_t lod_count, uint64_t* qw_out)
{
  return quant_weights_common(preds, n, num_points_in_lod, lod_count, nullptr, qw_out);
}

static int
lift_common(bool forward, const pccb200_predictor* preds, const uint64_t* qw, int32_t n,
            const uint32_t* num_points_in_lod, int32_t lod_count, int64_t* attrs, int32_t A)
{
  if (!preds || !qw || !num_points_in_lod || !attrs || n <= 0 || lod_count <= 0
      || (A != 1 && A != 3))
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    pccb200_predictor* dP = to_device(ex, preds, size_t(n));
    uint64_t* dQw = to_device(ex, qw, size_t(n));
    int64_t* dA = to_device(ex, attrs, size_t(n) * A);
    int rc = run_lift(ex, forward, dP, dQw, n, num_points_in_lod, lod_count, dA, A);
    if (rc != PCCB200_OK)
      return fail(rc, rc == PCCB200_ERR_UNSUPPORTED
                        ? "a predictor references its own level of detail"
                        : "numPointsInLod does not partition [0, n)");
    to_host(ex, attrs, dA, size_t(n) * A);
    return PCCB200_OK;
  });
}

int
pccb200_lift_forward(const pccb200_predictor* preds, const uint64_t* qw, int32_t n,
                     const uint32_t* num_points_in_lod, int32_t lod_count,
                     int64_t* attrs_inout, int32_t num_attrs)
{
  return lift_common(true, preds, qw, n, num_points_in_lod, lod_count, attrs_inout, num_attrs);
}

int
pccb200_lift_inverse(const pccb200_predictor* preds, const uint64_t* qw, int32_t n,
                     const uint32_t* num_points_in_lod, int32_t lod_count,
                     int64_t* attrs_inout, int32_t num_attrs)
{
  return lift_common(false, preds, qw, n, num_points_in_lod, lod_count, attrs_inout, num_attrs);
}

static int
lift_quant_common(bool forward, const pccb200_qpset* qpset, const int32_t* qpo,
                  const uint64_t* qw, int32_t n, const uint32_t* npl, int32_t lodCount,
                  int32_t numDetailLevels, int64_t* attrs, int32_t A, int32_t lcpEnabled,
                  int32_t* values, int8_t* lcp)
{
  if (!qpset || !qw || !npl || !attrs || !values || n <= 0 || (lcpEnabled && A == 3 && !lcp))
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    uint64_t* dQw = to_device(ex, qw, size_t(n));
    int32_t* dQpo = qpo ? to_device(ex, qpo, size_t(n) * 2) : nullptr;
    int64_t* dA = forward ? to_device(ex, attrs, size_t(n) * A) : ex.alloc<int64_t>(size_t(n) * A);
    int32_t* dV = forward ? ex.alloc<int32_t>(size_t(n) * A) : to_device(ex, values, size_t(n) * A);
    int rc = run_lift_quant(ex, forward, *qpset, dQpo, dQw, n, npl, lodCount, numDetailLevels, dA,
                            A, 0, A, lcpEnabled != 0, lcp, dV);
    if (rc != PCCB200_OK)
      return fail(rc, "invalid lifting quantisation parameters");
    to_host(ex, attrs, dA, size_t(n) * A);
    if (forward)
      to_host(ex, values, dV, size_t(n) * A);
    return PCCB200_OK;
  });
}

int
pccb200_lift_quantize(const pccb200_qpset* qpset, const int32_t* point_qp_offsets,
                      const uint64_t* qw, int32_t n, const uint32_t* num_points_in_lod,
                      int32_t lod_count, int32_t num_detail_levels, int64_t* attrs_inout,
                      int32_t num_attrs, int32_t lcp_enabled, int32_t* values_out,
                      int8_t* lcp_coeffs_out)
{
  return lift_quant_common(true, qpset, point_qp_offsets, qw, n, num_points_in_lod, lod_count,
                           num_detail_levels, attrs_inout, num_attrs, lcp_enabled, values_out,
                           lcp_coeffs_out);
}

int
pccb200_lift_dequantize(const pccb200_qpset* qpset, const int32_t* point_qp_offsets,
                        const uint64_t* qw, int32_t n, const uint32_t* num_points_in_lod,
                        int32_t lod_count, int32_t num_detail_levels, const int32_t* values_in,
                        int32_t num_attrs, const int8_t* lcp_coeffs, int64_t* attrs_out)
{
  return lift_quant_common(false, qpset, point_qp_offsets, qw, n, num_points_in_lod, lod_count,
                           num_detail_levels, attrs_out, num_attrs, lcp_coeffs != nullptr,
                           const_cast<int32_t*>(values_in), const_cast<int8_t*>(lcp_coeffs));
}

int
pccb200_lod_create(const pccb200_lod_params* params, const int32_t* xyz, int32_t n,
                   pccb200_lod_handle* handle_out)
{
  if (!params || !xyz || !handle_out || n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  *handle_out = nullptr;
  pccb200_lod_handle h = new (std::nothrow) pccb200_lod_handle_s();
  if (!h)
    return fail(PCCB200_ERR_NOMEM, "host allocation failed");
  h->params = *params;
  int rc = with_device([&](DeviceExec& ex) -> int {
    h->device = ctx().device;
    const size_t szP = (size_t(n) * sizeof(pccb200_predictor) + 255) & ~size_t(255);
    const size_t szQ = (size_t(n) * sizeof(uint64_t) + 255) & ~size_t(255);
    const size_t szI = (size_t(n) * sizeof(uint32_t) + 255) & ~size_t(255);
    PCC_CUDA_CHECK(cudaMalloc(&h->block, szP + szQ + szI));
    char* b = static_cast<char*>(h->block);
    h->st.preds = reinterpret_cast<pccb200_predictor*>(b);
    h->st.qw = reinterpret_cast<uint64_t*>(b + szP);
    h->st.idx = reinterpret_cast<uint32_t*>(b + szP + szQ);
    int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    int rc2 = lod_state_build(ex, *params, dXyz, n, h->st, false);
    if (rc2 != PCCB200_OK)
      return fail(rc2, "invalid LoD parameters");
    return PCCB200_OK;
  });
  if (rc != PCCB200_OK) {
    if (h->block)
      cudaFree(h->block);
    delete h;
    return rc;
  }
  *handle_out = h;
  return PCCB200_OK;
}

int
pccb200_lod_import(const pccb200_predictor* preds, const uint32_t* indexes, int32_t n,
                   const uint32_t* num_points_in_lod, int32_t lod_count,
                   int32_t num_detail_levels, const pccb200_lod_scalable* scal,
                   pccb200_lod_handle* handle_out)
{
  if (handle_out)
    *handle_out = nullptr;
  if (!preds || !indexes || !num_points_in_lod || !handle_out || n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  if (lod_count < 1 || lod_count > PCCB200_MAX_LODS)
    return fail(PCCB200_ERR_INVALID_ARG, "lod_count outside 1..PCCB200_MAX_LODS");
  for (int l = 0; l < lod_count; l++)
    if (num_points_in_lod[l] < (l ? num_points_in_lod[l - 1] : 1u))
      return fail(PCCB200_ERR_INVALID_ARG, "num_points_in_lod is not increasing");
  if (num_points_in_lod[lod_count - 1] != uint32_t(n))
    return fail(PCCB200_ERR_INVALID_ARG, "the last count of num_points_in_lod is not n");
  if (num_detail_levels < lod_count || num_detail_levels > PCCB200_MAX_LODS)
    return fail(PCCB200_ERR_INVALID_ARG, "num_detail_levels outside lod_count..PCCB200_MAX_LODS");
  if (scal && (scal->reserved != 0 || scal->min_geom_node_size_log2 < 0
               || scal->min_geom_node_size_log2 >= kScalableLevels
               || (scal->geom_num_points != 0 && scal->geom_num_points < n)))
    return fail(PCCB200_ERR_INVALID_ARG,
                "reserved not 0, min_geom_node_size_log2 out of range or geom_num_points < n");
  pccb200_lod_handle h = new (std::nothrow) pccb200_lod_handle_s();
  if (!h)
    return fail(PCCB200_ERR_NOMEM, "host allocation failed");
  h->params.num_detail_levels = num_detail_levels;
  h->imported = true;
  h->scalable = scal != nullptr;
  if (scal)
    h->scal = *scal;
  h->st.n = n;
  h->st.numDetailLevels = num_detail_levels;
  h->st.lodCount = lod_count;
  for (int l = 0; l < lod_count; l++)
    h->st.npl[l] = num_points_in_lod[l];
  int rc = with_device([&](DeviceExec& ex) -> int {
    h->device = ctx().device;
    const size_t szP = (size_t(n) * sizeof(pccb200_predictor) + 255) & ~size_t(255);
    const size_t szQ = (size_t(n) * sizeof(uint64_t) + 255) & ~size_t(255);
    const size_t szI = (size_t(n) * sizeof(uint32_t) + 255) & ~size_t(255);
    PCC_CUDA_CHECK(cudaMalloc(&h->block, szP + szQ + szI));
    char* b = static_cast<char*>(h->block);
    h->st.preds = reinterpret_cast<pccb200_predictor*>(b);
    h->st.qw = reinterpret_cast<uint64_t*>(b + szP);
    h->st.idx = reinterpret_cast<uint32_t*>(b + szP + szQ);
    ex.upload(h->st.preds, preds, size_t(n) * sizeof(pccb200_predictor));
    ex.upload(h->st.idx, indexes, size_t(n) * sizeof(uint32_t));
    if (run_lod_import_check(ex, h->st.preds, h->st.idx, n) != PCCB200_OK)
      return fail(PCCB200_ERR_INVALID_ARG,
                  "indexes is not a permutation of [0, n) or a predictor is malformed");
    return PCCB200_OK;
  });
  if (rc != PCCB200_OK) {
    if (h->block)
      cudaFree(h->block);
    delete h;
    return rc;
  }
  *handle_out = h;
  return PCCB200_OK;
}

void
pccb200_lod_destroy(pccb200_lod_handle handle)
{
  if (!handle)
    return;
  if (handle->block) {
    cudaSetDevice(handle->device);
    cudaFree(handle->block);
  }
  delete handle;
}

int
pccb200_lod_reusable(pccb200_lod_handle h, const pccb200_lod_params* p)
{
  if (!h || !p || h->imported)
    return 0;
  const pccb200_lod_params& a = h->params;
  // the order of AttributeLods::isReusable (tmc3/AttributeCommon.cpp:76-140)
  if (a.num_pred_nearest_neighbours != p->num_pred_nearest_neighbours
      || a.inter_lod_search_range != p->inter_lod_search_range
      || a.intra_lod_search_range != p->intra_lod_search_range
      || a.num_detail_levels != p->num_detail_levels)
    return 0;
  for (int k = 0; k < 3; k++)
    if (a.lod_neigh_bias[k] != p->lod_neigh_bias[k])
      return 0;
  if (a.lod_decimation_type != p->lod_decimation_type || a.dist2 != p->dist2)
    return 0;
  for (int l = 0; l < PCCB200_MAX_LODS; l++)
    if (a.lod_sampling_period[l] != p->lod_sampling_period[l])
      return 0;
  if (a.intra_lod_prediction_skip_layers != p->intra_lod_prediction_skip_layers
      || a.pred_weight_blending != p->pred_weight_blending
      || a.prediction_with_distribution != p->prediction_with_distribution)
    return 0;
  return 1;
}

int
pccb200_lod_info(pccb200_lod_handle h, int32_t* n_out, int32_t* lod_count_out,
                 uint32_t* num_points_in_lod_out)
{
  if (!h)
    return fail(PCCB200_ERR_INVALID_ARG, "null handle");
  if (n_out)
    *n_out = h->st.n;
  if (lod_count_out)
    *lod_count_out = h->st.lodCount;
  if (num_points_in_lod_out)
    for (int l = 0; l < PCCB200_MAX_LODS; l++)
      num_points_in_lod_out[l] = l < h->st.lodCount ? h->st.npl[l] : 0;
  return PCCB200_OK;
}

int
pccb200_attr_lift_encode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                             int32_t lcp_enabled, const int32_t* point_qp_offsets,
                             int32_t* attrs_inout, int32_t num_attrs, int32_t bitdepth,
                             int32_t* values_out, int8_t* lcp_coeffs_out)
{
  return attr_lift(true, false, nullptr, handle, qpset, lcp_enabled, point_qp_offsets, nullptr,
                   attrs_inout, num_attrs, bitdepth, nullptr, 0, values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                             int32_t lcp_enabled, const int32_t* point_qp_offsets,
                             int32_t* attrs_out, int32_t num_attrs, int32_t bitdepth,
                             const int32_t* values_in, const int8_t* lcp_coeffs)
{
  return attr_lift(false, false, nullptr, handle, qpset, lcp_enabled, point_qp_offsets, nullptr,
                   attrs_out, num_attrs, bitdepth, nullptr, 0, const_cast<int32_t*>(values_in),
                   const_cast<int8_t*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                         int32_t lcp_enabled, const int32_t* point_qp_offsets, const int32_t* xyz,
                         int32_t* attrs_inout, int32_t num_attrs, int32_t n, int32_t bitdepth,
                         int32_t* values_out, int8_t* lcp_coeffs_out)
{
  if (n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  const int64_t offs[2] = {0, n};
  return attr_lift(true, false, lod, nullptr, qpset, lcp_enabled, point_qp_offsets, xyz,
                   attrs_inout, num_attrs, bitdepth, offs, 1, values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                         int32_t lcp_enabled, const int32_t* point_qp_offsets, const int32_t* xyz,
                         int32_t* attrs_out, int32_t num_attrs, int32_t n, int32_t bitdepth,
                         const int32_t* values_in, const int8_t* lcp_coeffs)
{
  if (n <= 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  const int64_t offs[2] = {0, n};
  return attr_lift(false, false, lod, nullptr, qpset, lcp_enabled, point_qp_offsets, xyz,
                   attrs_out, num_attrs, bitdepth, offs, 1, const_cast<int32_t*>(values_in),
                   const_cast<int8_t*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_slices(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                const int32_t* xyz, int32_t* attrs_inout, int32_t num_attrs,
                                int32_t bitdepth, const int64_t* slice_offsets,
                                int32_t num_slices, int32_t* values_out, int8_t* lcp_coeffs_out)
{
  return attr_lift(true, false, lod, nullptr, qpset, lcp_enabled, point_qp_offsets, xyz,
                   attrs_inout, num_attrs, bitdepth, slice_offsets, num_slices, values_out,
                   lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_slices(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                const int32_t* xyz, int32_t* attrs_out, int32_t num_attrs,
                                int32_t bitdepth, const int64_t* slice_offsets,
                                int32_t num_slices, const int32_t* values_in,
                                const int8_t* lcp_coeffs)
{
  return attr_lift(false, false, lod, nullptr, qpset, lcp_enabled, point_qp_offsets, xyz,
                   attrs_out, num_attrs, bitdepth, slice_offsets, num_slices,
                   const_cast<int32_t*>(values_in), const_cast<int8_t*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_slices_dev(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                    int32_t lcp_enabled, const int32_t* d_point_qp_offsets,
                                    const int32_t* d_xyz, int32_t* d_attrs_inout,
                                    int32_t num_attrs, int32_t bitdepth,
                                    const int64_t* slice_offsets, int32_t num_slices,
                                    int32_t* d_values_out, int8_t* lcp_coeffs_out)
{
  return attr_lift(true, true, lod, nullptr, qpset, lcp_enabled, d_point_qp_offsets, d_xyz,
                   d_attrs_inout, num_attrs, bitdepth, slice_offsets, num_slices, d_values_out,
                   lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_slices_dev(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                    int32_t lcp_enabled, const int32_t* d_point_qp_offsets,
                                    const int32_t* d_xyz, int32_t* d_attrs_out, int32_t num_attrs,
                                    int32_t bitdepth, const int64_t* slice_offsets,
                                    int32_t num_slices, const int32_t* d_values_in,
                                    const int8_t* lcp_coeffs)
{
  return attr_lift(false, true, lod, nullptr, qpset, lcp_enabled, d_point_qp_offsets, d_xyz,
                   d_attrs_out, num_attrs, bitdepth, slice_offsets, num_slices,
                   const_cast<int32_t*>(d_values_in), const_cast<int8_t*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_multi(const pccb200_lod_params* lod, int32_t num_sets,
                               const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                               const int32_t* xyz, int32_t n, int32_t* const* attrs_inout,
                               const int32_t* num_attrs, const int32_t* bitdepths,
                               int32_t* const* values_out, int8_t* const* lcp_coeffs_out)
{
  return attr_lift_multi(true, false, 1, &lod, num_sets, qpsets, lcp_enabled, &xyz, &n,
                         attrs_inout, num_attrs, bitdepths, values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_multi(const pccb200_lod_params* lod, int32_t num_sets,
                               const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                               const int32_t* xyz, int32_t n, int32_t* const* attrs_out,
                               const int32_t* num_attrs, const int32_t* bitdepths,
                               const int32_t* const* values_in, const int8_t* const* lcp_coeffs)
{
  return attr_lift_multi(false, false, 1, &lod, num_sets, qpsets, lcp_enabled, &xyz, &n,
                         attrs_out, num_attrs, bitdepths, const_cast<int32_t* const*>(values_in),
                         const_cast<int8_t* const*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_multi_dev(const pccb200_lod_params* lod, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                   const int32_t* d_xyz, int32_t n, int32_t* const* d_attrs_inout,
                                   const int32_t* num_attrs, const int32_t* bitdepths,
                                   int32_t* const* d_values_out, int8_t* const* lcp_coeffs_out)
{
  return attr_lift_multi(true, true, 1, &lod, num_sets, qpsets, lcp_enabled, &d_xyz, &n,
                         d_attrs_inout, num_attrs, bitdepths, d_values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_multi_dev(const pccb200_lod_params* lod, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                   const int32_t* d_xyz, int32_t n, int32_t* const* d_attrs_out,
                                   const int32_t* num_attrs, const int32_t* bitdepths,
                                   const int32_t* const* d_values_in,
                                   const int8_t* const* lcp_coeffs)
{
  return attr_lift_multi(false, true, 1, &lod, num_sets, qpsets, lcp_enabled, &d_xyz, &n,
                         d_attrs_out, num_attrs, bitdepths,
                         const_cast<int32_t* const*>(d_values_in),
                         const_cast<int8_t* const*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_multi_batch(int32_t num_units, const pccb200_lod_params* const* lods,
                                     int32_t num_sets, const pccb200_qpset* const* qpsets,
                                     const int32_t* lcp_enabled, const int32_t* const* xyz,
                                     const int32_t* n, int32_t* const* attrs_inout,
                                     const int32_t* num_attrs, const int32_t* bitdepths,
                                     int32_t* const* values_out, int8_t* const* lcp_coeffs_out)
{
  return attr_lift_multi(true, false, num_units, lods, num_sets, qpsets, lcp_enabled, xyz, n,
                         attrs_inout, num_attrs, bitdepths, values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_multi_batch(int32_t num_units, const pccb200_lod_params* const* lods,
                                     int32_t num_sets, const pccb200_qpset* const* qpsets,
                                     const int32_t* lcp_enabled, const int32_t* const* xyz,
                                     const int32_t* n, int32_t* const* attrs_out,
                                     const int32_t* num_attrs, const int32_t* bitdepths,
                                     const int32_t* const* values_in,
                                     const int8_t* const* lcp_coeffs)
{
  return attr_lift_multi(false, false, num_units, lods, num_sets, qpsets, lcp_enabled, xyz, n,
                         attrs_out, num_attrs, bitdepths, const_cast<int32_t* const*>(values_in),
                         const_cast<int8_t* const*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_multi_batch_dev(int32_t num_units, const pccb200_lod_params* const* lods,
                                         int32_t num_sets, const pccb200_qpset* const* qpsets,
                                         const int32_t* lcp_enabled, const int32_t* const* d_xyz,
                                         const int32_t* n, int32_t* const* d_attrs_inout,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         int32_t* const* d_values_out,
                                         int8_t* const* lcp_coeffs_out)
{
  return attr_lift_multi(true, true, num_units, lods, num_sets, qpsets, lcp_enabled, d_xyz, n,
                         d_attrs_inout, num_attrs, bitdepths, d_values_out, lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_multi_batch_dev(int32_t num_units, const pccb200_lod_params* const* lods,
                                         int32_t num_sets, const pccb200_qpset* const* qpsets,
                                         const int32_t* lcp_enabled, const int32_t* const* d_xyz,
                                         const int32_t* n, int32_t* const* d_attrs_out,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         const int32_t* const* d_values_in,
                                         const int8_t* const* lcp_coeffs)
{
  return attr_lift_multi(false, true, num_units, lods, num_sets, qpsets, lcp_enabled, d_xyz, n,
                         d_attrs_out, num_attrs, bitdepths,
                         const_cast<int32_t* const*>(d_values_in),
                         const_cast<int8_t* const*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_scalable(int32_t num_units, const pccb200_lod_params* const* lods,
                                  const pccb200_lod_scalable* scals, int32_t num_sets,
                                  const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                  const int32_t* const* xyz, const int32_t* n,
                                  int32_t* const* attrs_inout, const int32_t* num_attrs,
                                  const int32_t* bitdepths, int32_t* const* values_out,
                                  int8_t* const* lcp_coeffs_out)
{
  return attr_lift_scalable(true, false, num_units, lods, scals, num_sets, qpsets, lcp_enabled,
                            xyz, n, attrs_inout, num_attrs, bitdepths, values_out,
                            lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_scalable(int32_t num_units, const pccb200_lod_params* const* lods,
                                  const pccb200_lod_scalable* scals, int32_t num_sets,
                                  const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                  const int32_t* const* xyz, const int32_t* n,
                                  int32_t* const* attrs_out, const int32_t* num_attrs,
                                  const int32_t* bitdepths, const int32_t* const* values_in,
                                  const int8_t* const* lcp_coeffs)
{
  return attr_lift_scalable(false, false, num_units, lods, scals, num_sets, qpsets, lcp_enabled,
                            xyz, n, attrs_out, num_attrs, bitdepths,
                            const_cast<int32_t* const*>(values_in),
                            const_cast<int8_t* const*>(lcp_coeffs));
}

int
pccb200_attr_lift_encode_scalable_dev(int32_t num_units, const pccb200_lod_params* const* lods,
                                      const pccb200_lod_scalable* scals, int32_t num_sets,
                                      const pccb200_qpset* const* qpsets,
                                      const int32_t* lcp_enabled, const int32_t* const* d_xyz,
                                      const int32_t* n, int32_t* const* d_attrs_inout,
                                      const int32_t* num_attrs, const int32_t* bitdepths,
                                      int32_t* const* d_values_out, int8_t* const* lcp_coeffs_out)
{
  return attr_lift_scalable(true, true, num_units, lods, scals, num_sets, qpsets, lcp_enabled,
                            d_xyz, n, d_attrs_inout, num_attrs, bitdepths, d_values_out,
                            lcp_coeffs_out);
}

int
pccb200_attr_lift_decode_scalable_dev(int32_t num_units, const pccb200_lod_params* const* lods,
                                      const pccb200_lod_scalable* scals, int32_t num_sets,
                                      const pccb200_qpset* const* qpsets,
                                      const int32_t* lcp_enabled, const int32_t* const* d_xyz,
                                      const int32_t* n, int32_t* const* d_attrs_out,
                                      const int32_t* num_attrs, const int32_t* bitdepths,
                                      const int32_t* const* d_values_in,
                                      const int8_t* const* lcp_coeffs)
{
  return attr_lift_scalable(false, true, num_units, lods, scals, num_sets, qpsets, lcp_enabled,
                            d_xyz, n, d_attrs_out, num_attrs, bitdepths,
                            const_cast<int32_t* const*>(d_values_in),
                            const_cast<int8_t* const*>(lcp_coeffs));
}

//----------------------------------------------------------------------------
// spherical coordinates (spherical.cuh)

static int
spherical_common(const int32_t* origin, const int32_t* theta, int32_t numTheta,
                 const int32_t* weight, const int32_t* minPos, const int32_t* xyz, int64_t n,
                 int32_t* out, int32_t* bbox)
{
  if (!origin || !theta || !xyz || !out || !bbox || numTheta < 1 || n < 0
      || n > int64_t(INT32_MAX) / 3)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    const int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    const int32_t* dTheta = to_device(ex, theta, size_t(numTheta));
    int32_t* dOut = ex.alloc<int32_t>(size_t(n) * 3);
    run_xyz_to_rpl(ex, origin, dTheta, numTheta, dXyz, n, dOut, bbox, minPos, weight);
    to_host(ex, out, dOut, size_t(n) * 3);
    return PCCB200_OK;
  });
}

int
pccb200_xyz_to_rpl(const int32_t laser_origin[3], const int32_t* laser_theta, int32_t num_theta,
                   const int32_t* xyz, int64_t n, int32_t* rpl_out, int32_t bbox_out[6])
{
  return spherical_common(laser_origin, laser_theta, num_theta, nullptr, nullptr, xyz, n,
                          rpl_out, bbox_out);
}

int
pccb200_attr_spherical_positions(const int32_t laser_origin[3], const int32_t* laser_theta,
                                 int32_t num_theta, const int32_t axis_weight[3],
                                 const int32_t* min_pos, const int32_t* xyz, int64_t n,
                                 int32_t* pos_out, int32_t bbox_out[6])
{
  if (!axis_weight)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return spherical_common(laser_origin, laser_theta, num_theta, axis_weight, min_pos, xyz, n,
                          pos_out, bbox_out);
}

int
pccb200_offset_and_scale(const int32_t min_pos[3], const int32_t axis_weight[3],
                         int32_t* pos_inout, int64_t n)
{
  if (!min_pos || !axis_weight || !pos_inout || n < 0 || n > int64_t(INT32_MAX) / 3)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    int32_t* dPos = to_device(ex, pos_inout, size_t(n) * 3);
    OffsetScaleFn os;
    for (int k = 0; k < 3; k++) {
      os.minPos[k] = min_pos[k];
      os.weight[k] = axis_weight[k];
    }
    os.pos = dPos;
    ex.foreach(n, os);
    to_host(ex, pos_inout, dPos, size_t(n) * 3);
    return PCCB200_OK;
  });
}

//----------------------------------------------------------------------------
// symbol preparation for the entropy coder (symbols.cuh)

static void
symbols_to_host(DeviceExec& ex, const int32_t* dRuns, const int32_t* dValues, const uint8_t* dCtx,
                int count, int A, int32_t* runs, int32_t* values, uint8_t* ctx)
{
  to_host(ex, runs, dRuns, size_t(count));
  to_host(ex, values, dValues, size_t(count) * A);
  if (ctx && A == 3)
    to_host(ex, ctx, dCtx, size_t(count));
}

int
pccb200_coeff_symbols(const int32_t* coeffs, int32_t num_attrs, int32_t n,
                      int32_t* zero_runs_out, int32_t* values_out, uint8_t* ctx_out,
                      int32_t* count_out, int32_t* tail_run_out)
{
  if (!coeffs || !zero_runs_out || !values_out || !count_out || !tail_run_out || n <= 0
      || (num_attrs != 1 && num_attrs != 3))
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    const int A = num_attrs;
    const int32_t* dCoef = to_device(ex, coeffs, size_t(n) * A);
    int32_t* dRuns = ex.alloc<int32_t>(size_t(n));
    int32_t* dValues = ex.alloc<int32_t>(size_t(n) * A);
    uint8_t* dCtx = ex.alloc<uint8_t>(size_t(n));
    int count = 0, tail = 0;
    run_coeff_symbols(ex, dCoef, n, A, n, dRuns, dValues, dCtx, &count, &tail);
    symbols_to_host(ex, dRuns, dValues, dCtx, count, A, zero_runs_out, values_out, ctx_out);
    *count_out = count;
    *tail_run_out = tail;
    return PCCB200_OK;
  });
}

int
pccb200_attr_raht_encode_symbols(const pccb200_raht_params* params, const pccb200_qpset* qpset,
                                 const int32_t* point_qp_offsets, const int32_t* xyz,
                                 int32_t* attrs_inout, int32_t num_attrs, int32_t n,
                                 int32_t bitdepth, int32_t* zero_runs_out, int32_t* values_out,
                                 uint8_t* ctx_out, int32_t* count_out, int32_t* tail_run_out)
{
  const int64_t offs[2] = {0, n};
  int rc = check_slices(params, qpset, xyz, attrs_inout, values_out, num_attrs, bitdepth, offs, 1);
  if (rc != PCCB200_OK)
    return rc;
  if (!zero_runs_out || !count_out || !tail_run_out || num_attrs == 2)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    const int A = num_attrs;
    // the unit is staged here: its coefficients stay on the device
    RahtUnit u;
    u.n = n;
    u.xyz = to_device(ex, xyz, size_t(n) * 3);
    u.qpo = point_qp_offsets ? to_device(ex, point_qp_offsets, size_t(n) * 2) : nullptr;
    u.dev = true;
    u.numSets = 1;
    u.qs[0] = qpset;
    u.A[0] = A;
    u.bitdepth[0] = bitdepth;
    u.attrs[0] = to_device(ex, attrs_inout, size_t(n) * A);
    u.coef[0] = ex.alloc<int32_t>(size_t(n) * A);
    u.coefStride[0] = n;
    int rc2 = code_units(ex, true, *params, &u, 1);
    if (rc2 != PCCB200_OK)
      return rc2;
    const int32_t* dCoef = u.coef[0];
    to_host(ex, attrs_inout, u.attrs[0], size_t(n) * A);
    int32_t* dRuns = ex.alloc<int32_t>(size_t(n));
    int32_t* dValues = ex.alloc<int32_t>(size_t(n) * A);
    uint8_t* dCtx = ex.alloc<uint8_t>(size_t(n));
    int count = 0, tail = 0;
    run_coeff_symbols(ex, dCoef, n, A, n, dRuns, dValues, dCtx, &count, &tail);
    symbols_to_host(ex, dRuns, dValues, dCtx, count, A, zero_runs_out, values_out, ctx_out);
    *count_out = count;
    *tail_run_out = tail;
    return PCCB200_OK;
  });
}

//----------------------------------------------------------------------------
// estimateDist2 (dist2.cuh)

int
pccb200_estimate_dist2(const int32_t* xyz, int32_t n, int32_t sampling_period,
                       int32_t search_range, float percentile_estimate, int32_t* shift_bits_out)
{
  if (!xyz || !shift_bits_out || n < 0 || sampling_period < 1 || search_range < 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  if (n < 2) {
    *shift_bits_out = 0;
    return PCCB200_OK;
  }
  return with_device([&](DeviceExec& ex) -> int {
    const int32_t* dXyz = to_device(ex, xyz, size_t(n) * 3);
    const int s = run_estimate_dist2(ex, dXyz, n, sampling_period, search_range,
                                     percentile_estimate);
    if (s < 0)
      return fail(PCCB200_ERR_INVALID_ARG, "percentile outside [0, 1)");
    *shift_bits_out = s;
    return PCCB200_OK;
  });
}

//----------------------------------------------------------------------------
// the other two quantisation-weight derivations (lifting.cuh)

int
pccb200_quant_weights_fixed(const pccb200_predictor* preds, int32_t n,
                            const uint32_t* num_points_in_lod, int32_t lod_count,
                            const int32_t neigh_weight[3], uint64_t* qw_out)
{
  if (!neigh_weight)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return quant_weights_common(preds, n, num_points_in_lod, lod_count, neigh_weight, qw_out);
}

int
pccb200_quant_weights_scalable(const uint32_t* num_points_in_lod, int32_t lod_count,
                               int64_t num_points, int32_t min_geom_node_size_log2, int32_t n,
                               uint64_t* qw_out)
{
  if (!num_points_in_lod || !qw_out || n <= 0 || lod_count <= 0 || num_points < 0)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return with_device([&](DeviceExec& ex) -> int {
    uint64_t* dQw = ex.alloc<uint64_t>(n);
    int rc = run_quant_weights_scalable(ex, num_points_in_lod, lod_count, uint64_t(num_points),
                                        min_geom_node_size_log2, n, dQw);
    if (rc != PCCB200_OK)
      return fail(rc, "numPointsInLod does not partition [0, n)");
    to_host(ex, qw_out, dQw, size_t(n));
    return PCCB200_OK;
  });
}

//----------------------------------------------------------------------------
// recolouring (recolour.cuh)

void
pccb200_recolour_params_default(pccb200_recolour_params* p)
{
  if (!p)
    return;
  // tmc3/TMC3.cpp:1500-1551
  p->dist_offset_fwd = 4.;
  p->dist_offset_bwd = 4.;
  p->max_geometry_dist2_fwd = 1000.;
  p->max_geometry_dist2_bwd = 1000.;
  p->max_attribute_dist2_fwd = 1000.;
  p->max_attribute_dist2_bwd = 1000.;
  p->search_range = 1;
  p->num_neighbours_fwd = 8;
  p->num_neighbours_bwd = 1;
  p->use_dist_weighted_avg_fwd = 1;
  p->use_dist_weighted_avg_bwd = 1;
  p->skip_avg_if_identical_source_point_present_fwd = 1;
  p->skip_avg_if_identical_source_point_present_bwd = 0;
  p->reserved = 0;
}

int
pccb200_recolour(const pccb200_recolour_params* params, const int32_t* source_xyz,
                 const int32_t* source_attrs, int32_t num_attrs, int32_t n_source,
                 double source_to_target_scale, const int32_t tgt_to_src_offset[3],
                 const int32_t* target_xyz, int32_t n_target, int32_t bitdepth,
                 int32_t* target_attrs_out)
{
  if (!params || !source_xyz || !source_attrs || !tgt_to_src_offset || !target_xyz
      || !target_attrs_out || n_source <= 0 || n_target <= 0 || (num_attrs != 1 && num_attrs != 3))
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  // the other ranges are checked on the device path (recolour_run)
  std::vector<RecolourUnit> units(1);
  RecolourUnit& u = units[0];
  u.nSrc = n_source;
  u.nTgt = n_target;
  u.srcXyz = source_xyz;
  u.tgtXyz = target_xyz;
  u.scale = source_to_target_scale;
  for (int k = 0; k < 3; k++)
    u.off[k] = tgt_to_src_offset[k];
  u.numSets = 1;
  u.sets[0] = RecolourSet{source_attrs, num_attrs, bitdepth, nullptr, target_attrs_out};
  return code_recolour(*params, units, false);
}

int
pccb200_recolour_multi(const pccb200_recolour_params* params, int32_t num_sets,
                       const int32_t* source_xyz, int32_t n_source,
                       const int32_t* const* source_attrs, const int32_t* num_attrs,
                       const int32_t* bitdepths, double source_to_target_scale,
                       const int32_t tgt_to_src_offset[3], const int32_t* target_xyz,
                       int32_t n_target, int32_t* const* target_attrs_out)
{
  return recolour_multi(false, params, num_sets, 1, &source_xyz, &n_source, source_attrs,
                        num_attrs, bitdepths, &source_to_target_scale, tgt_to_src_offset,
                        &target_xyz, &n_target, target_attrs_out);
}

int
pccb200_recolour_multi_dev(const pccb200_recolour_params* params, int32_t num_sets,
                           const int32_t* d_source_xyz, int32_t n_source,
                           const int32_t* const* d_source_attrs, const int32_t* num_attrs,
                           const int32_t* bitdepths, double source_to_target_scale,
                           const int32_t tgt_to_src_offset[3], const int32_t* d_target_xyz,
                           int32_t n_target, int32_t* const* d_target_attrs_out)
{
  return recolour_multi(true, params, num_sets, 1, &d_source_xyz, &n_source, d_source_attrs,
                        num_attrs, bitdepths, &source_to_target_scale, tgt_to_src_offset,
                        &d_target_xyz, &n_target, d_target_attrs_out);
}

int
pccb200_recolour_multi_batch(const pccb200_recolour_params* params, int32_t num_sets,
                             int32_t num_units, const int32_t* const* source_xyz,
                             const int32_t* n_source, const int32_t* const* source_attrs,
                             const int32_t* num_attrs, const int32_t* bitdepths,
                             const double* source_to_target_scale,
                             const int32_t* tgt_to_src_offsets, const int32_t* const* target_xyz,
                             const int32_t* n_target, int32_t* const* target_attrs_out)
{
  return recolour_multi(false, params, num_sets, num_units, source_xyz, n_source, source_attrs,
                        num_attrs, bitdepths, source_to_target_scale, tgt_to_src_offsets,
                        target_xyz, n_target, target_attrs_out);
}

int
pccb200_recolour_multi_batch_dev(const pccb200_recolour_params* params, int32_t num_sets,
                                 int32_t num_units, const int32_t* const* d_source_xyz,
                                 const int32_t* n_source, const int32_t* const* d_source_attrs,
                                 const int32_t* num_attrs, const int32_t* bitdepths,
                                 const double* source_to_target_scale,
                                 const int32_t* tgt_to_src_offsets,
                                 const int32_t* const* d_target_xyz, const int32_t* n_target,
                                 int32_t* const* d_target_attrs_out)
{
  return recolour_multi(true, params, num_sets, num_units, d_source_xyz, n_source, d_source_attrs,
                        num_attrs, bitdepths, source_to_target_scale, tgt_to_src_offsets,
                        d_target_xyz, n_target, d_target_attrs_out);
}

// the reference-exact recolouring: nanoflann's trees and search, std::sort's
// list order (recolour.cuh, kRecolourRefExact)

int
pccb200_recolour_exact(const pccb200_recolour_params* params, const int32_t* source_xyz,
                       const int32_t* source_attrs, int32_t num_attrs, int32_t n_source,
                       double source_to_target_scale, const int32_t tgt_to_src_offset[3],
                       const int32_t* target_xyz, int32_t n_target, int32_t bitdepth,
                       int32_t* target_attrs_out)
{
  if (!params || !source_xyz || !source_attrs || !tgt_to_src_offset || !target_xyz
      || !target_attrs_out)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer or bad size");
  return recolour_multi(false, params, 1, 1, &source_xyz, &n_source, &source_attrs, &num_attrs,
                        &bitdepth, &source_to_target_scale, tgt_to_src_offset, &target_xyz,
                        &n_target, &target_attrs_out, kRecolourRefExact);
}

int
pccb200_recolour_exact_multi_batch(const pccb200_recolour_params* params, int32_t num_sets,
                                   int32_t num_units, const int32_t* const* source_xyz,
                                   const int32_t* n_source, const int32_t* const* source_attrs,
                                   const int32_t* num_attrs, const int32_t* bitdepths,
                                   const double* source_to_target_scale,
                                   const int32_t* tgt_to_src_offsets,
                                   const int32_t* const* target_xyz, const int32_t* n_target,
                                   int32_t* const* target_attrs_out)
{
  return recolour_multi(false, params, num_sets, num_units, source_xyz, n_source, source_attrs,
                        num_attrs, bitdepths, source_to_target_scale, tgt_to_src_offsets,
                        target_xyz, n_target, target_attrs_out, kRecolourRefExact);
}

int
pccb200_recolour_exact_multi_batch_dev(const pccb200_recolour_params* params, int32_t num_sets,
                                       int32_t num_units, const int32_t* const* d_source_xyz,
                                       const int32_t* n_source,
                                       const int32_t* const* d_source_attrs,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       const double* source_to_target_scale,
                                       const int32_t* tgt_to_src_offsets,
                                       const int32_t* const* d_target_xyz,
                                       const int32_t* n_target, int32_t* const* d_target_attrs_out)
{
  return recolour_multi(true, params, num_sets, num_units, d_source_xyz, n_source, d_source_attrs,
                        num_attrs, bitdepths, source_to_target_scale, tgt_to_src_offsets,
                        d_target_xyz, n_target, d_target_attrs_out, kRecolourRefExact);
}

//----------------------------------------------------------------------------
// predicting-transform decoder (pred_pipeline.cuh)

int
pccb200_attr_pred_decode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                             const pccb200_pred_params* pred, const int32_t quant_neigh_weight[3],
                             const int32_t* point_qp_offsets, const int8_t* icp_coeffs,
                             const int32_t* values_in, int32_t num_attrs, int32_t bitdepth,
                             int32_t* attrs_out)
{
  if (!handle || !quant_neigh_weight || !values_in || !attrs_out
      || check_pred_set(qpset, pred, num_attrs, bitdepth) != PCCB200_OK)
    return fail(PCCB200_ERR_INVALID_ARG, "null pointer, bad size or bad parameters");
  if (handle->scalable)
    return fail(PCCB200_ERR_UNSUPPORTED, "scalable lifting levels of detail");
  std::vector<PredCallUnit> units(1);
  PredCallUnit& cu = units[0];
  cu.n = handle->st.n;
  cu.qpo = point_qp_offsets;
  cu.handle = handle;
  for (int k = 0; k < 3; k++)
    cu.pu.quantNeighWeight[k] = quant_neigh_weight[k];
  cu.pu.numSets = 1;
  cu.pu.sets[0] = PredSet{num_attrs, bitdepth, qpset, *pred, values_in, icp_coeffs, attrs_out};
  return code_pred(false, units);
}

int
pccb200_attr_pred_decode_multi_batch(
  int32_t num_units, const pccb200_lod_params* const* lods, const int32_t* quant_neigh_weight,
  int32_t num_sets, const pccb200_qpset* const* qpsets, const pccb200_pred_params* pred,
  const int32_t* num_attrs, const int32_t* bitdepths, const int32_t* const* xyz, const int32_t* n,
  const int32_t* const* point_qp_offsets, const int32_t* const* values_in,
  const int8_t* const* icp_coeffs, int32_t* const* attrs_out)
{
  return attr_pred_multi(false, num_units, lods, quant_neigh_weight, num_sets, qpsets, pred,
                         num_attrs, bitdepths, xyz, n, point_qp_offsets, values_in, icp_coeffs,
                         attrs_out);
}

int
pccb200_attr_pred_decode_multi_batch_dev(
  int32_t num_units, const pccb200_lod_params* const* lods, const int32_t* quant_neigh_weight,
  int32_t num_sets, const pccb200_qpset* const* qpsets, const pccb200_pred_params* pred,
  const int32_t* num_attrs, const int32_t* bitdepths, const int32_t* const* d_xyz,
  const int32_t* n, const int32_t* const* d_point_qp_offsets, const int32_t* const* d_values_in,
  const int8_t* const* icp_coeffs, int32_t* const* d_attrs_out)
{
  return attr_pred_multi(true, num_units, lods, quant_neigh_weight, num_sets, qpsets, pred,
                         num_attrs, bitdepths, d_xyz, n, d_point_qp_offsets, d_values_in,
                         icp_coeffs, d_attrs_out);
}

}  // extern "C"
