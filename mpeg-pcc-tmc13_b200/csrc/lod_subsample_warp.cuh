// lod_subsample_warp.cuh — distance subsampling (subsampleByDistance,
// tmc3/PCCTMC3Common.h:1984-2085) as a warp-cooperative dataflow over cells
// (device only).  Same decisions as SubsampleDistanceFn in lod_core.cuh (the
// host-testable definition):
//   * k_cell_neighbours: one thread per (cell, neighbour offset) resolves the
//     19 neighbour cells by binary search — geometry only, fully parallel;
//   * k_subsample_cells: one warp per cell in Morton ticket order.  A cell's
//     latency is what bounds a level (cells wait for the decisions of earlier
//     neighbour cells), so the cell's first points are fetched before the
//     wait; then 19 lanes poll the 16-byte records of the neighbour cells:
//     (x, y, z, state) of the cell's retained point, written with ONE aligned
//     16-byte store and read with one 16-byte load (a single transaction
//     each, as in the status + value words of a decoupled look-back scan), so
//     that the hop from a cell to the next is one L2 round trip: no release
//     fence on the producer's side, no second dependent load on the
//     consumer's; the cell's points are tested one after the other, all
//     neighbours at once (ballot).
#pragma once

#include "lod_core.cuh"

namespace pccb200 {

struct SubsampleCellsArgs {
  Voxels v;
  const uint32_t* input;
  const int32_t* cellFirst;
  int nCells;
  int shiftBits0;
  int* decision;
  uint8_t* keep;
  const int32_t* order;  // wavefront schedule: ticket t runs cell order[t] (null: Morton order)
  int32_t* nb;  // nCells * 19 neighbour cell indices (or -1)
  int4* decPos;  // per cell: (x, y, z) of its retained point, w = kCellRec* (zeroed before the launch)
};

constexpr int kCellRecUndecided = 0, kCellRecNone = 1, kCellRecPoint = 2;

__device__ __forceinline__ int4
ld_cell_rec(const int4* p)
{
  int4 v;
  asm volatile("ld.relaxed.gpu.global.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void
st_cell_rec(int4* p, int x, int y, int z, int w)
{
  asm volatile("st.relaxed.gpu.global.v4.s32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(x), "r"(y),
               "r"(z), "r"(w)
               : "memory");
}

__global__ void __launch_bounds__(256)
k_cell_neighbours(const SubsampleCellsArgs a)
{
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (tid >= int64_t(a.nCells) * 19)
    return;
  const int c = int(tid / 19);
  const int n = int(tid - int64_t(c) * 19) + 1;
  const uint8_t kOff[20] = {7,  3,  5,  6,  12, 10, 17, 20, 34, 33,
                            4,  2,  1,  24, 40, 48, 32, 16, 8,  0};
  const int sb3 = 3 * (a.shiftBits0 + 1);
  const int atlasBit = sb3 + 21 < 63 ? sb3 + 21 : 63;
  const int64_t code0 = a.v.code[a.input[a.cellFirst[c]]];
  const int64_t cell = code0 >> sb3;
  const int64_t atlasId = code0 >> atlasBit;
  const uint64_t base = morton3d_add(uint64_t(cell), ~uint64_t(0));
  const int64_t nc = int64_t(morton3d_add(base, kOff[n]));
  int q = -1;
  if ((nc >> 21) == atlasId) {
    q = find_cell(a.v.code, a.input, a.cellFirst, a.nCells, sb3, nc);
    if (q >= c || (q >= 0 && (a.v.code[a.input[a.cellFirst[q]]] >> atlasBit) != atlasId))
      q = -1;
  }
  a.nb[tid] = q;
}

__global__ void __launch_bounds__(256)
k_subsample_cells(const SubsampleCellsArgs a, unsigned long long* ticket)
{
  const int lane = threadIdx.x & 31;
  const int64_t radius2 = int64_t(3) << (a.shiftBits0 << 1);
  for (;;) {
    unsigned long long t = 0;
    if (lane == 0)
      t = atomicAdd(ticket, 1ull);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= (unsigned long long)a.nCells)
      return;
    const int c = a.order ? a.order[t] : int(t);
    const int q = lane < 19 ? a.nb[size_t(c) * 19 + lane] : -1;
    const int i0 = a.cellFirst[c], i1 = a.cellFirst[c + 1];
    // the first two points of the cell (the same in every lane), before the wait
    int32_t pa[3] = {0, 0, 0}, pb[3] = {0, 0, 0};
    {
      const uint32_t ia = a.input[i0];
      const uint32_t ib = i0 + 1 < i1 ? a.input[i0 + 1] : ia;
      const int32_t* p = &a.v.pos[size_t(ia) * 3];
      const int32_t* r = &a.v.pos[size_t(ib) * 3];
      pa[0] = p[0];
      pa[1] = p[1];
      pa[2] = p[2];
      pb[0] = r[0];
      pb[1] = r[1];
      pb[2] = r[2];
    }
    // retained point of this lane's neighbour cell (if any)
    bool have = false;
    int32_t np[3] = {0, 0, 0};
    if (q >= 0) {
      int4 r = ld_cell_rec(&a.decPos[q]);
      while (r.w == kCellRecUndecided) {
        __nanosleep(32);
        r = ld_cell_rec(&a.decPos[q]);
      }
      if (r.w == kCellRecPoint) {
        np[0] = r.x;
        np[1] = r.y;
        np[2] = r.z;
        have = true;
      }
    }
    int chosen = kCellNone;
    for (int i = i0; i < i1; i++) {
      int32_t pp[3];
      if (i == i0) {
        pp[0] = pa[0], pp[1] = pa[1], pp[2] = pa[2];
      } else if (i == i0 + 1) {
        pp[0] = pb[0], pp[1] = pb[1], pp[2] = pb[2];
      } else {
        const int32_t* p = &a.v.pos[size_t(a.input[i]) * 3];
        pp[0] = p[0], pp[1] = p[1], pp[2] = p[2];
      }
      const bool hit = have && norm2_3(np, pp) <= radius2;
      const bool found = __ballot_sync(0xffffffffu, hit) != 0;
      if (!found) {
        chosen = i;
        // the retained point's position travels with the decision
        if (lane == 0) {
          st_cell_rec(&a.decPos[c], pp[0], pp[1], pp[2], kCellRecPoint);
          a.keep[i] = 1;
        }
        for (int r = i + 1 + lane; r < i1; r += 32)
          a.keep[r] = 0;
        break;
      }
      if (lane == 0)
        a.keep[i] = 0;
    }
    if (chosen == kCellNone && lane == 0)
      st_cell_rec(&a.decPos[c], 0, 0, 0, kCellRecNone);
  }
}

// Dependency level of every cell (1 + the highest level among the earlier
// neighbour cells it waits for): geometry only.  Claimed in Morton order, the
// cells of a long chain sit in the ticket window while cells that could run
// wait to be claimed (the time per hop grows with the size of the level);
// sorted by level
// (wavefront order) a cell is normally ready when a warp takes it.  One thread
// per cell, 32 consecutive cells per ticket, the polling loop uniform over the
// warp (as k_block_levels in raht_wave.cuh).
__global__ void __launch_bounds__(256)
k_cell_levels(const int32_t* __restrict__ nb, const int nCells, int* lv, int64_t* key,
              int32_t* val, unsigned long long* ticket)
{
  const int lane = threadIdx.x & 31;
  for (;;) {
    unsigned long long base = 0;
    if (lane == 0)
      base = atomicAdd(ticket, 32ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base >= (unsigned long long)nCells)
      return;
    const int c = int(base) + lane;
    const bool active = c < nCells;
    int q[19];
#pragma unroll
    for (int i = 0; i < 19; i++)
      q[i] = active ? nb[size_t(c) * 19 + i] : -1;
    bool done = !active;
    while (__any_sync(0xffffffffu, !done)) {
      bool progress = false;
      if (!done) {
        int m = 0;
        bool ready = true;
#pragma unroll
        for (int i = 0; i < 19; i++)
          if (q[i] >= 0) {
            int v;
            asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(lv + q[i]) : "memory");
            if (!v)
              ready = false;
            else
              m = v > m ? v : m;
          }
        if (ready) {
          m++;
          asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(lv + c), "r"(m) : "memory");
          key[c] = m;
          val[c] = c;
          done = true;
          progress = true;
        }
      }
      if (!__any_sync(0xffffffffu, progress))
        __nanosleep(40);
    }
  }
}

}  // namespace pccb200
