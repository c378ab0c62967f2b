// morton_sort.cuh — Morton key generation and a stable LSD radix sort of
// (int64 key, int32 index) pairs.
//
// Replaces mortonAddr + std::sort over MortonCodeWithIndex, whose comparison
// falls back to the point index on equal codes (i.e. a stable sort by code):
//   tmc3/PCCMath.h:605-626, tmc3/PCCTMC3Common.h:176-191,
//   tmc3/AttributeEncoder.cpp:1316-1321, tmc3/AttributeDecoder.cpp:623-628.
//
// One pass per 8 key bits; only as many passes as the widest key needs
// (3 x coordinate bits; the OR of all keys is reduced while they are
// generated).  Each pass: per-tile digit histograms -> exclusive scan in
// digit-major order -> stable scatter.  Inside a tile every warp ranks a
// contiguous run of keys with __match_any_sync, so loads are coalesced and
// equal digits keep their input order.
#pragma once

#include "exec_cuda.cuh"
#include "pcc_arith.cuh"

namespace pccb200 {

constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;
constexpr int kSortTile = kSortThreads * kSortItems;  // 4096 keys per CTA
constexpr int kSortWarps = kSortThreads / 32;
constexpr uint64_t kSignFlip = uint64_t(1) << 63;     // signed -> unsigned order

__global__ void __launch_bounds__(256)
k_morton_keys(const int32_t* __restrict__ xyz, int64_t n, int64_t* __restrict__ keys,
              int32_t* __restrict__ idx, unsigned long long* __restrict__ orAll)
{
  unsigned long long acc = 0;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    int64_t k = morton_addr(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    keys[i] = k;
    idx[i] = int32_t(i);
    acc |= (unsigned long long)k;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1)
    acc |= __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc)
    atomicOr(orAll, acc);
}

__global__ void __launch_bounds__(kSortThreads)
k_radix_hist(const int64_t* __restrict__ keys, int64_t n, int shift, int numTiles,
             int* __restrict__ hist)
{
  __shared__ int sHist[256];
  sHist[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = int64_t(blockIdx.x) * kSortTile;
#pragma unroll
  for (int j = 0; j < kSortItems; j++) {
    int64_t i = base + j * kSortThreads + threadIdx.x;
    if (i < n) {
      unsigned d = unsigned(((uint64_t(keys[i]) ^ kSignFlip) >> shift) & 0xff);
      atomicAdd(&sHist[d], 1);
    }
  }
  __syncthreads();
  hist[threadIdx.x * numTiles + blockIdx.x] = sHist[threadIdx.x];
}

// generic exclusive scan of an int array: tile sums, scan of the tile sums by
// one CTA (k_scan_tiles), tile scans with their offsets
__global__ void __launch_bounds__(kTileThreads)
k_scan_sum(const int* __restrict__ in, int64_t n, int* __restrict__ tileSum)
{
  const int64_t base = int64_t(blockIdx.x) * kTile + threadIdx.x * kTileItems;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kTileItems; j++)
    if (base + j < n)
      c += in[base + j];
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
    tileSum[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kTileThreads)
k_scan_apply(int* __restrict__ data, int64_t n, const int* __restrict__ tileOffset)
{
  const int64_t base = int64_t(blockIdx.x) * kTile + threadIdx.x * kTileItems;
  int v[kTileItems];
  int c = 0;
#pragma unroll
  for (int j = 0; j < kTileItems; j++) {
    v[j] = base + j < n ? data[base + j] : 0;
    c += v[j];
  }
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
  int off = tileOffset[blockIdx.x] + x - c;
  for (int w = 0; w < (threadIdx.x >> 5); w++)
    off += sWarp[w];
#pragma unroll
  for (int j = 0; j < kTileItems; j++)
    if (base + j < n) {
      data[base + j] = off;
      off += v[j];
    }
}

__global__ void __launch_bounds__(kSortThreads)
k_radix_scatter(const int64_t* __restrict__ keysIn, const int32_t* __restrict__ valsIn,
                int64_t* __restrict__ keysOut, int32_t* __restrict__ valsOut, int64_t n,
                int shift, int numTiles, const int* __restrict__ offsets)
{
  __shared__ int sCount[kSortWarps][256];
  for (int i = threadIdx.x; i < kSortWarps * 256; i += kSortThreads)
    (&sCount[0][0])[i] = 0;
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t base = int64_t(blockIdx.x) * kSortTile + warp * (32 * kSortItems);
  const unsigned ltMask = (1u << lane) - 1;

  int64_t key[kSortItems];
  int32_t val[kSortItems];
  int rank[kSortItems];
#pragma unroll
  for (int j = 0; j < kSortItems; j++) {
    int64_t i = base + j * 32 + lane;
    const bool valid = i < n;
    key[j] = valid ? keysIn[i] : 0;
    val[j] = valid ? valsIn[i] : 0;
    unsigned d = unsigned(((uint64_t(key[j]) ^ kSignFlip) >> shift) & 0xff);
    // lanes past the end vote in a bucket of their own (0x100) so that they
    // never disturb the ranks of real keys
    unsigned peers = __match_any_sync(0xffffffffu, valid ? d : 0x100u);
    int before = sCount[warp][d];
    rank[j] = before + __popc(peers & ltMask);
    __syncwarp();
    if (valid && (peers & ltMask) == 0)
      sCount[warp][d] = before + __popc(peers);
    __syncwarp();
  }
  __syncthreads();

  // exclusive prefix over the warps of this tile, per digit
  {
    int d = threadIdx.x;  // kSortThreads == 256 digits
    int run = offsets[d * numTiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kSortWarps; w++) {
      int c = sCount[w][d];
      sCount[w][d] = run;
      run += c;
    }
  }
  __syncthreads();

#pragma unroll
  for (int j = 0; j < kSortItems; j++) {
    int64_t i = base + j * 32 + lane;
    if (i < n) {
      unsigned d = unsigned(((uint64_t(key[j]) ^ kSignFlip) >> shift) & 0xff);
      int64_t dst = int64_t(sCount[warp][d]) + rank[j];
      keysOut[dst] = key[j];
      valsOut[dst] = val[j];
    }
  }
}

// out[i*outStride + outOff + k] = in[order[i]*A + k]  (one attribute of several
// into the interleaved rows of a multi-attribute pass)
__global__ void __launch_bounds__(256)
k_gather_rows_strided(const int32_t* __restrict__ in, const int32_t* __restrict__ order,
                      int64_t n, int A, int32_t* __restrict__ out, int outStride, int outOff)
{
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    int64_t src = order[i];
    for (int k = 0; k < A; k++)
      out[i * outStride + outOff + k] = in[src * A + k];
  }
}

// out[order[i]*A + k] = clip(in[i*inStride + inOff + k], 0, clipMax)
__global__ void __launch_bounds__(256)
k_scatter_rows_clip_strided(const int32_t* __restrict__ in, int inStride, int inOff,
                            const int32_t* __restrict__ order, int64_t n, int A,
                            int32_t clipMax, int32_t* __restrict__ out)
{
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    int64_t dst = order[i];
    for (int k = 0; k < A; k++) {
      int32_t v = in[i * inStride + inOff + k];
      v = v < 0 ? 0 : (v > clipMax ? clipMax : v);
      out[dst * A + k] = v;
    }
  }
}

inline unsigned
grid_for(int64_t n, int numSMs)
{
  int64_t b = (n + 255) / 256;
  int64_t cap = int64_t(numSMs) * 16;
  return unsigned(b < 1 ? 1 : (b > cap ? cap : b));
}

// Stable LSD radix sort of (int64 key, int32 value) pairs on the low
// 8 * passes key bits.  The pairs ping-pong between (keysA, valsA) and
// (keysB, valsB); *keysRes / *valsRes say where the result landed.
inline void
device_radix_sort_pairs(DeviceExec& ex, int64_t* keysA, int32_t* valsA, int64_t* keysB,
                        int32_t* valsB, int64_t n, int passes, int64_t** keysRes,
                        int32_t** valsRes)
{
  cudaStream_t st = ex.stream;
  const int numTiles = int((n + kSortTile - 1) / kSortTile);
  const int64_t histLen = int64_t(256) * numTiles;
  int* hist = ex.alloc<int>(histLen);
  const int scanTiles = int((histLen + kTile - 1) / kTile);
  int* tileSums = ex.alloc<int>(scanTiles);

  int64_t* kin = keysA;
  int32_t* vin = valsA;
  int64_t* kout = keysB;
  int32_t* vout = valsB;
  for (int p = 0; p < passes; p++) {
    const int shift = 8 * p;
    DeviceExec::Scope sc(ex);
    k_radix_hist<<<numTiles, kSortThreads, 0, st>>>(kin, n, shift, numTiles, hist);
    k_scan_sum<<<scanTiles, kTileThreads, 0, st>>>(hist, histLen, tileSums);
    k_scan_tiles<<<1, 1024, 0, st>>>(tileSums, scanTiles, nullptr);
    k_scan_apply<<<scanTiles, kTileThreads, 0, st>>>(hist, histLen, tileSums);
    k_radix_scatter<<<numTiles, kSortThreads, 0, st>>>(kin, vin, kout, vout, n, shift,
                                                       numTiles, hist);
    g_launchCount += 5;
    int64_t* tk = kin;
    kin = kout;
    kout = tk;
    int32_t* tv = vin;
    vin = vout;
    vout = tv;
  }
  PCC_CUDA_CHECK(cudaGetLastError());
  *keysRes = kin;
  *valsRes = vin;
}

// Sorts n points; keysOut / orderOut are device buffers of n entries.
// Uses the executor's arena for scratch.  One synchronising read-back (the OR
// of all keys) decides the number of passes.
inline void
device_morton_sort(DeviceExec& ex, const int32_t* dXyz, int64_t n, int64_t* keysOut,
                   int32_t* orderOut)
{
  if (n <= 0)
    return;
  ex.phase(kPhaseSort);
  cudaStream_t st = ex.stream;
  int64_t* keysTmp = ex.alloc<int64_t>(n);
  int32_t* valsTmp = ex.alloc<int32_t>(n);
  unsigned long long* dOr = ex.alloc<unsigned long long>(1);
  PCC_CUDA_CHECK(cudaMemsetAsync(dOr, 0, sizeof(unsigned long long), st));

  // the pass count is not known yet, so generate into the "A" buffers and
  // let the parity of the pass count decide where the result lands
  {
    DeviceExec::Scope sc(ex);
    k_morton_keys<<<grid_for(n, ex.numSMs), 256, 0, st>>>(dXyz, n, keysOut, orderOut, dOr);
  }
  g_launchCount++;
  unsigned long long hOr = 0;
  ex.download(&hOr, dOr, sizeof(hOr));
  int bits = 64 - (hOr ? __builtin_clzll(hOr) : 64);
  int passes = (bits + 7) / 8;
  if (passes == 0)
    return;  // all keys zero: already sorted, order = identity

  int64_t* kres = nullptr;
  int32_t* vres = nullptr;
  device_radix_sort_pairs(ex, keysOut, orderOut, keysTmp, valsTmp, n, passes, &kres, &vres);
  if (kres != keysOut) {
    PCC_CUDA_CHECK(cudaMemcpyAsync(keysOut, kres, n * sizeof(int64_t),
                                   cudaMemcpyDeviceToDevice, st));
    PCC_CUDA_CHECK(cudaMemcpyAsync(orderOut, vres, n * sizeof(int32_t),
                                   cudaMemcpyDeviceToDevice, st));
  }
}

inline void
DeviceExec::morton_sort(const int32_t* xyz, int64_t n, int64_t* keys, int32_t* order)
{
  device_morton_sort(*this, xyz, n, keys, order);
}

inline const int32_t*
DeviceExec::cell_wave_order(const int32_t* nb, int nCells)
{
  int* lv = alloc<int>(size_t(nCells) + 2);
  zero(lv, (size_t(nCells) + 2) * sizeof(int));
  unsigned long long* tk = reinterpret_cast<unsigned long long*>(alloc<int64_t>(1));
  zero(tk, sizeof(unsigned long long));
  int64_t* keyA = alloc<int64_t>(size_t(nCells));
  int64_t* keyB = alloc<int64_t>(size_t(nCells));
  int32_t* valA = alloc<int32_t>(size_t(nCells));
  int32_t* valB = alloc<int32_t>(size_t(nCells));
  int64_t blocks = (int64_t(nCells) + 255) / 256;
  const int64_t cap = int64_t(numSMs) * 8;
  k_cell_levels<<<unsigned(blocks > cap ? cap : blocks), 256, 0, stream>>>(nb, nCells, lv, keyA, valA, tk);
  g_launchCount++;
  int64_t* kres;
  int32_t* vres;
  device_radix_sort_pairs(*this, keyA, valA, keyB, valB, nCells, 3, &kres, &vres);
  return vres;
}

// in-place exclusive prefix sum of n ints (the scan of the radix sort's histograms)
inline void
DeviceExec::exclusive_scan(int* data, int64_t n)
{
  if (n <= 0)
    return;
  const int scanTiles = int((n + kTile - 1) / kTile);
  int* tileSums = alloc<int>(scanTiles);
  Scope sc(*this);
  k_scan_sum<<<scanTiles, kTileThreads, 0, stream>>>(data, n, tileSums);
  k_scan_tiles<<<1, 1024, 0, stream>>>(tileSums, scanTiles, nullptr);
  k_scan_apply<<<scanTiles, kTileThreads, 0, stream>>>(data, n, tileSums);
  g_launchCount += 3;
  PCC_CUDA_CHECK(cudaGetLastError());
}

}  // namespace pccb200
