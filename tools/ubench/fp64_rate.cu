// micro-benchmark: fp64 DFMA and DMMA (m8n8k4, m16n8k16) issue rate / latency, SHFL and LDS cost for one warp and for a full GPU (H100)
#include <cstdio>
#include <cuda_runtime.h>
__global__ void dfma_kernel(double* out, int iters, long long* cyc) {
  double acc[32]; double a = out[threadIdx.x & 31], b = 1.0000001;
#pragma unroll
  for (int i = 0; i < 32; i++) acc[i] = a + i;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = fma(acc[i], b, a);
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) s += acc[i];
  out[blockIdx.x*blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void dfma_dep_kernel(double* out, int iters, long long* cyc) {
  double acc = out[threadIdx.x & 31], b = 1.0000001;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 32; i++) acc = fma(acc, b, 0.5);
  }
  long long t1 = clock64();
  out[blockIdx.x*blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void shfl_kernel(double* out, int iters, long long* cyc) {
  double v = out[threadIdx.x & 31]; double acc[16];
#pragma unroll
  for (int i = 0; i < 16; i++) acc[i] = i;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 16; i++) acc[i] += __shfl_sync(0xffffffffu, v, i);
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) s += acc[i];
  out[blockIdx.x*blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void lds_kernel(double* out, int iters, long long* cyc) {
  __shared__ double sm[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = i;
  __syncthreads();
  double acc[16];
#pragma unroll
  for (int i = 0; i < 16; i++) acc[i] = i;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 16; i += 2) { double2 b = *reinterpret_cast<double2*>(&sm[(it & 31)*32 + i]); acc[i] += b.x; acc[i+1] += b.y; }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) s += acc[i];
  out[blockIdx.x*blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void rsqrt_kernel(double* out, int iters, long long* cyc) {
  double v = out[threadIdx.x & 31] + 2.0;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) { v = rsqrt(v) + 1.5; }
  long long t1 = clock64();
  out[blockIdx.x*blockDim.x + threadIdx.x] = v;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void dmma_kernel(double* out, int iters, long long* cyc, int nacc) {
  double a0 = out[threadIdx.x & 31] + 1.0, b0 = 1.0000001;
  double c[16][2];
#pragma unroll
  for (int i = 0; i < 16; i++) { c[i][0] = i; c[i][1] = -i; }
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 16; i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a0), "d"(b0));
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) s += c[i][0] + c[i][1];
  out[blockIdx.x*blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void dmma16_kernel(double* out, int iters, long long* cyc) {   // mma.sync m16n8k16 f64 (sm_90), 4 independent
  double a0 = 1e-3*(threadIdx.x & 31), b0 = 1e-3;
  double c[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) c[i][j] = i - j;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 4; i++)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4,%4,%4,%4,%4,%4,%4}, {%5,%5,%5,%5}, {%0,%1,%2,%3};"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a0), "d"(b0));
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x*blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void dmma_dep_kernel(double* out, int iters, long long* cyc) {
  double a0 = out[threadIdx.x & 31] + 1.0, b0 = 1.0000001, c0 = 0, c1 = 0;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 16; i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a0), "d"(b0));
  }
  long long t1 = clock64();
  out[blockIdx.x*blockDim.x + threadIdx.x] = c0 + c1;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
int main() {
  double* d; long long* c; cudaMalloc(&d, 1 << 24); cudaMemset(d, 0, 1 << 24); cudaMalloc(&c, 8);
  long long h; const int it = 2000;
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int cfg = 0; cfg < 3; cfg++) {
    int blocks = cfg == 0 ? 1 : sms*(cfg == 1 ? 1 : 4), threads = cfg == 0 ? 32 : (cfg == 1 ? 128 : 256);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    dfma_kernel<<<blocks, threads>>>(d, it, c); cudaDeviceSynchronize();
    cudaEventRecord(e0); dfma_kernel<<<blocks, threads>>>(d, it, c); cudaEventRecord(e1); cudaDeviceSynchronize();
    cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); cudaEventElapsedTime(&ms, e0, e1);
    printf("dfma indep  blocks %4d x %3d thr: %.2f cyc per warp-DFMA (warp 0), chip %.2f TFLOP/s\n", blocks, threads, (double)h/(it*32), 2.0*blocks*threads*it*32/(ms*1e-3)/1e12);
  }
  dfma_dep_kernel<<<1, 32>>>(d, it, c); cudaDeviceSynchronize(); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); printf("dfma dependent chain: %.2f cyc latency\n", (double)h/(it*32));
  shfl_kernel<<<1, 32>>>(d, it, c); cudaDeviceSynchronize(); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); printf("shfl(double)+dadd, 1 warp: %.2f cyc each\n", (double)h/(it*16));
  lds_kernel<<<1, 32>>>(d, it, c); cudaDeviceSynchronize(); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); printf("lds.128 bcast + 2 dadd, 1 warp: %.2f cyc each\n", (double)h/(it*8));
  rsqrt_kernel<<<1, 32>>>(d, it, c); cudaDeviceSynchronize(); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); printf("rsqrt(double)+dadd dependent: %.2f cyc\n", (double)h/it);
  for (int cfg = 0; cfg < 3; cfg++) {
    int blocks = cfg == 0 ? 1 : sms*(cfg == 1 ? 1 : 4), threads = cfg == 0 ? 32 : (cfg == 1 ? 128 : 256);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    dmma_kernel<<<blocks, threads>>>(d, it, c, 16); cudaDeviceSynchronize();
    cudaEventRecord(e0); dmma_kernel<<<blocks, threads>>>(d, it, c, 16); cudaEventRecord(e1); cudaDeviceSynchronize();
    cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); cudaEventElapsedTime(&ms, e0, e1);
    printf("dmma m8n8k4 indep blocks %4d x %3d thr: %.2f cyc per warp-DMMA (warp 0), chip %.2f TFLOP/s\n", blocks, threads, (double)h/(it*16), 2.0*256*(double)blocks*(threads/32)*it*16/(ms*1e-3)/1e12);
  }
  for (int cfg = 1; cfg < 3; cfg++) {
    int blocks = sms*(cfg == 1 ? 1 : 4), threads = cfg == 1 ? 128 : 256;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    dmma16_kernel<<<blocks, threads>>>(d, it, c); cudaDeviceSynchronize();
    cudaEventRecord(e0); dmma16_kernel<<<blocks, threads>>>(d, it, c); cudaEventRecord(e1); cudaDeviceSynchronize();
    cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); cudaEventElapsedTime(&ms, e0, e1);
    printf("dmma m16n8k16 indep blocks %4d x %3d thr: %.2f cyc per warp-DMMA (warp 0), chip %.2f TFLOP/s\n", blocks, threads, (double)h/(it*4), 4096.0*(double)blocks*(threads/32)*it*4/(ms*1e-3)/1e12);
  }
  dmma_dep_kernel<<<1, 32>>>(d, it, c); cudaDeviceSynchronize(); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost); printf("dmma dependent chain: %.2f cyc latency\n", (double)h/(it*16));
  return 0;
}
