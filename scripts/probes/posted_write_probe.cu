// Probe (not part of the product): bandwidth of a kernel's own stores into pinned host memory (posted PCIe writes) for
// different store shapes. 4096 rows of 1600 bytes (case33 observations without padding) per launch.
//   nvcc -O2 -gencode arch=compute_90a,code=sm_90a -o scripts/probes/posted_write_probe scripts/probes/posted_write_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)
constexpr int ROWS = 4096, ROW16 = 100;             // 100 x 16 B per row
// mode 0: 8 lanes per row (128 B per row and instruction), the 4 rows of a warp are different rows (the env kernel's shape)
// mode 1: 32 lanes per row (512 contiguous bytes per instruction), a warp handles its 4 rows one after another
// mode 2: like 0 but 16 lanes per row (256 B)
// mode 3: like 1, but each lane stores 2 x 16 B back to back (1 KB contiguous per warp and pair of instructions)
__global__ void k(double2* dst, int mode, int rows_per_block) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const double2 v = make_double2(threadIdx.x, blockIdx.x);
  const int row0 = blockIdx.x * rows_per_block;
  for (int r = warp * 4; r < rows_per_block; r += nw * 4) {
    if (mode == 0) {
      const int row = row0 + r + (lane >> 3);
      if (row < ROWS && r + (lane >> 3) < rows_per_block) for (int c = lane & 7; c < ROW16; c += 8) dst[size_t(row) * ROW16 + c] = v;
    } else if (mode == 2) {
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + r + 2 * h + (lane >> 4);
        if (row < ROWS && r + 2 * h + (lane >> 4) < rows_per_block) for (int c = lane & 15; c < ROW16; c += 16) dst[size_t(row) * ROW16 + c] = v;
      }
    } else if (mode == 1) {
      for (int q = 0; q < 4; ++q) {
        const int row = row0 + r + q;
        if (row < ROWS && r + q < rows_per_block) for (int c = lane; c < ROW16; c += 32) dst[size_t(row) * ROW16 + c] = v;
      }
    } else {
      for (int q = 0; q < 4; ++q) {
        const int row = row0 + r + q;
        if (row < ROWS && r + q < rows_per_block)
          for (int c = 2 * lane; c < ROW16; c += 64) { dst[size_t(row) * ROW16 + c] = v; dst[size_t(row) * ROW16 + c + 1] = v; }
      }
    }
  }
}
int main() {
  const size_t bytes = size_t(ROWS) * ROW16 * 16;
  double2 *host, *dev;
  CK(cudaMallocHost(&host, bytes)); CK(cudaMalloc(&dev, bytes));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int reps = 30;
  for (int blocks : {132, 264, 528}) {
    const int rpb = (ROWS + blocks - 1) / blocks;
    for (int mode = 0; mode < 4; ++mode) {
      for (int tgt = 0; tgt < 2; ++tgt) {
        double2* d = tgt ? dev : host;
        for (int pass = 0; pass < 2; ++pass) {
          CK(cudaEventRecord(e0));
          for (int r = 0; r < reps; ++r) k<<<blocks, 256>>>(d, mode, rpb);
          CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
          float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
          if (pass) printf("blocks %3d mode %d -> %s: %7.1f us  %6.1f GB/s\n", blocks, mode, tgt ? "HBM " : "host", 1e3 * ms / reps, bytes * reps / (ms * 1e6));
        }
      }
    }
  }
  return 0;
}
