// PCIe probe for the ROI ingest (k_ingest): what the link gives to (1) the copy engine, (2) a zero-copy kernel reading a
// contiguous pinned buffer, (3) the ROI pattern of configs[3] (128 bodies x one 608 B x 202 row colour rectangle + one 256 B
// x 128 row depth rectangle out of 640x480 frames) with several launch shapes, (4) 256 cudaMemcpy2DAsync calls.
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o scripts/probes/pcie_probe scripts/probes/pcie_probe.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

template <int INFLIGHT>
__global__ void k_contig(const uint4* __restrict__ src, uint4* dst, size_t n) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += INFLIGHT * stride) {
    uint4 v[INFLIGHT];
#pragma unroll
    for (int u = 0; u < INFLIGHT; ++u) if (i + u * stride < n) v[u] = __ldg(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < INFLIGHT; ++u) if (i + u * stride < n) dst[i + u * stride] = v[u];
  }
}

struct Rect { const unsigned char* src; unsigned char* dst; unsigned pitch, row_bytes, rows; };

template <int INFLIGHT>
__global__ void k_roi(const Rect* rects, int rects_per_body, int ctas_per_body) {
  const int body = blockIdx.x / ctas_per_body, part = blockIdx.x % ctas_per_body;
  for (int q = 0; q < rects_per_body; ++q) {
    const Rect r = rects[body * rects_per_body + q];
    const int per_row = int(r.row_bytes >> 4);
    const int total = per_row * int(r.rows);
    const int step = blockDim.x * ctas_per_body;
    for (int c0 = part * blockDim.x + threadIdx.x; c0 < total; c0 += INFLIGHT * step) {
      uint4 v[INFLIGHT];
#pragma unroll
      for (int u = 0; u < INFLIGHT; ++u) {
        const int c = c0 + u * step;
        if (c < total) { const int row = c / per_row, k = c - row * per_row; v[u] = __ldg(reinterpret_cast<const uint4*>(r.src + size_t(row) * r.pitch) + k); }
      }
#pragma unroll
      for (int u = 0; u < INFLIGHT; ++u) {
        const int c = c0 + u * step;
        if (c < total) { const int row = c / per_row, k = c - row * per_row; reinterpret_cast<uint4*>(r.dst + size_t(row) * r.pitch)[k] = v[u]; }
      }
    }
  }
}

int main() {
  const int n_bodies = 128;
  const size_t cbytes = 640 * 480 * 3, dbytes = 640 * 480 * 2;
  const size_t total = n_bodies * (cbytes + dbytes);
  unsigned char *h, *d;
  CK(cudaHostAlloc(&h, total, cudaHostAllocDefault));
  CK(cudaMalloc(&d, total));
  for (size_t i = 0; i < total; i += 4096) h[i] = (unsigned char)i;
  cudaStream_t s; CK(cudaStreamCreate(&s));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float ms;
  auto report = [&](const char* name, double bytes, float ms, int reps) { printf("%-64s %8.3f ms  %7.2f GB/s\n", name, ms / reps, bytes * reps / (ms * 1e6)); };
  const int reps = 10;
  {  // (1) copy engine, 64 MiB
    const size_t n = 64u << 20;
    CK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(e0, s));
    for (int r = 0; r < reps; ++r) CK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
    report("copy engine, one 64 MiB cudaMemcpyAsync", double(n), ms, reps);
    const size_t m = 20u << 20;
    CK(cudaEventRecord(e0, s));
    for (int r = 0; r < reps; ++r) CK(cudaMemcpyAsync(d, h, m, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
    report("copy engine, one 20 MiB cudaMemcpyAsync", double(m), ms, reps);
  }
  {  // (2) zero-copy contiguous
    const size_t n = (64u << 20) / 16;
    const int grids[3] = {132, 264, 528};  // 1, 2, 4 CTAs per SM of an H100 SXM
    for (int g : grids) {
      k_contig<4><<<g, 256, 0, s>>>(reinterpret_cast<const uint4*>(h), reinterpret_cast<uint4*>(d), n);
      CK(cudaEventRecord(e0, s));
      for (int r = 0; r < reps; ++r) k_contig<4><<<g, 256, 0, s>>>(reinterpret_cast<const uint4*>(h), reinterpret_cast<uint4*>(d), n);
      CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      char name[96]; snprintf(name, sizeof name, "zero-copy kernel, contiguous 64 MiB, %d CTAs x 256, 4 x 16 B/thread", g);
      report(name, double(n * 16), ms, reps);
    }
    k_contig<8><<<296, 256, 0, s>>>(reinterpret_cast<const uint4*>(h), reinterpret_cast<uint4*>(d), n);
    CK(cudaEventRecord(e0, s));
    for (int r = 0; r < reps; ++r) k_contig<8><<<296, 256, 0, s>>>(reinterpret_cast<const uint4*>(h), reinterpret_cast<uint4*>(d), n);
    CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
    report("zero-copy kernel, contiguous 64 MiB, 296 CTAs x 256, 8 x 16 B/thread", double(n * 16), ms, reps);
  }
  // (3) ROI pattern
  for (int variant = 0; variant < 3; ++variant) {
    // variant 0: as configs[3] (608 B x 202, 256 B x 128); 1: colour rows widened to 128 B multiples and 128 B aligned; 2: full-width rows
    std::vector<Rect> rects;
    double bytes = 0;
    for (int b = 0; b < n_bodies; ++b) {
      unsigned char* hc = h + size_t(b) * (cbytes + dbytes); unsigned char* hd = hc + cbytes;
      unsigned char* dc = d + size_t(b) * (cbytes + dbytes); unsigned char* dd = dc + cbytes;
      const int x0 = 208 + 16 * (b % 5), y0 = 130 + (b % 7);
      Rect c, dp;
      if (variant == 0) { c = {hc + y0 * 1920 + x0 * 3, dc + y0 * 1920 + x0 * 3, 1920, 608, 202}; dp = {hd + (y0 + 30) * 1280 + (x0 + 40) * 2, dd + (y0 + 30) * 1280 + (x0 + 40) * 2, 1280, 256, 128}; }
      else if (variant == 1) { const size_t off = (size_t(y0) * 1920 + x0 * 3) / 128 * 128, offd = (size_t(y0 + 30) * 1280 + (x0 + 40) * 2) / 128 * 128;
        c = {hc + off, dc + off, 1920, 768, 202}; dp = {hd + offd, dd + offd, 1280, 384, 128}; }
      else { c = {hc + y0 * 1920, dc + y0 * 1920, 1920, 1920, 202}; dp = {hd + (y0 + 30) * 1280, dd + (y0 + 30) * 1280, 1280, 1280, 128}; }
      rects.push_back(c); rects.push_back(dp);
      bytes += double(c.row_bytes) * c.rows + double(dp.row_bytes) * dp.rows;
    }
    Rect* drects; CK(cudaMalloc(&drects, rects.size() * sizeof(Rect)));
    CK(cudaMemcpy(drects, rects.data(), rects.size() * sizeof(Rect), cudaMemcpyHostToDevice));
    const char* vn[3] = {"ROI 608 B x 202 + 256 B x 128", "ROI 128 B aligned rows (768 B x 202 + 384 B x 128)", "ROI full-width rows (1920 B x 202 + 1280 B x 128)"};
    for (int shape = 0; shape < 5; ++shape) {
      const int ctas = shape == 0 ? 1 : shape == 1 ? 2 : shape == 2 ? 4 : shape == 3 ? 1 : 2;
      const int threads = shape <= 2 ? 256 : 1024;
      auto launch = [&]() {
        if (shape == 4) k_roi<8><<<n_bodies * ctas, threads, 0, s>>>(drects, 2, ctas);
        else k_roi<4><<<n_bodies * ctas, threads, 0, s>>>(drects, 2, ctas);
      };
      launch();
      CK(cudaEventRecord(e0, s));
      for (int r = 0; r < reps; ++r) launch();
      CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      char name[128]; snprintf(name, sizeof name, "%s, %d CTA/body x %d, %d in flight", vn[variant], ctas, threads, shape == 4 ? 8 : 4);
      report(name, bytes, ms, reps);
    }
    if (variant == 0) {  // (4) copy engine, 2-D copies
      CK(cudaEventRecord(e0, s));
      for (int r = 0; r < reps; ++r)
        for (const Rect& q : rects) CK(cudaMemcpy2DAsync(q.dst, q.pitch, q.src, q.pitch, q.row_bytes, q.rows, cudaMemcpyHostToDevice, s));
      CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      report("copy engine, 256 cudaMemcpy2DAsync (same rectangles)", bytes, ms, reps);
    }
    CK(cudaFree(drects));
  }
  return 0;
}
