// Micro-benchmark of the warp-cooperative truncating pseudo-inverse (abrb_coop.cuh): cycles per pass, alone on an SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/dbg/coop_time tools/dbg/coop_time.cu
//   tools/dbg/coop_time tools/dbg/slow_A.bin     (KD x N = 6 x 6 matrices A of UR5 states on the pinv route, doubles)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../abr_control_b200/csrc/abrb_coop.cuh"
using namespace abrb;

struct Slot { static __device__ __forceinline__ int at(int r, int k) { return 12 + r * 6 + k; } };
struct Layout { static constexpr int kY = 0, kZ = 6; };

// one warp per CTA; `per_warp` waiting lanes per warp (1 .. 32); exchange area layout: [0,12) y z, [12,48) A
__global__ void bench(const double *A, int n_states, int per_warp, long long *cycles, double *out) {
  __shared__ double xch[48 * 32];
  const int lane = threadIdx.x;
  const int s = (blockIdx.x * per_warp + lane) % n_states;
  const bool slow = lane < per_warp;
  for (int i = 0; i < 12; ++i) xch[i * 32 + lane] = 0.1 * (i + 1);
  for (int i = 0; i < 36; ++i) xch[(12 + i) * 32 + lane] = A[(size_t)s * 36 + i];
  __syncwarp();
  const unsigned mask = __ballot_sync(0xffffffffu, slow);
  const long long t0 = clock64();
  coop_pinv_warp<double, 6, 6, Slot, Layout>(mask, xch, xch, lane, 1e-4, true);
  const long long t1 = clock64();
  __syncwarp();
  if (lane == 0) cycles[blockIdx.x] = t1 - t0;
  out[blockIdx.x * 32 + lane] = xch[lane];
}

int main(int argc, char **argv) {
  FILE *f = fopen(argc > 1 ? argv[1] : "tools/dbg/slow_A.bin", "rb");
  if (!f) return 1;
  std::vector<double> A;
  double buf[36];
  while (fread(buf, sizeof(double), 36, f) == 36) A.insert(A.end(), buf, buf + 36);
  fclose(f);
  const int n = (int)(A.size() / 36);
  double *dA, *dout;
  long long *dc;
  cudaMalloc(&dA, A.size() * 8);
  cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice);
  const int grid = 132;
  cudaMalloc(&dc, grid * 8);
  cudaMalloc(&dout, grid * 32 * 8);
  for (int per_warp : {1, 4, 5, 6, 10, 32}) {  // five states per pass (six-lane groups)
    bench<<<grid, 32>>>(dA, n, per_warp, dc, dout);
    bench<<<grid, 32>>>(dA, n, per_warp, dc, dout);
    cudaDeviceSynchronize();
    std::vector<long long> c(grid);
    cudaMemcpy(c.data(), dc, grid * 8, cudaMemcpyDeviceToHost);
    long long mn = c[0], mx = c[0], sum = 0;
    for (auto v : c) { mn = v < mn ? v : mn; mx = v > mx ? v : mx; sum += v; }
    printf("waiting lanes per warp %2d: cycles per call  min %lld  mean %lld  max %lld   (%s)\n", per_warp, mn, sum / grid, mx,
           cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
