// stockham.cu -- host side of stockham.cuh: the twiddle tables shared by the shared-memory FFT kernels.
#include <math.h>
#include <mutex>
#include <vector>
#include "stockham.cuh"

const float2 *af_twiddle_table(int log2n) {
    static std::mutex mu;
    static float2 *cache[64][32];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || log2n < 1 || log2n > 24) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    if (cache[dev][log2n]) return cache[dev][log2n];
    const size_t n = (size_t)1 << log2n;
    std::vector<float2> h(2 * n + 1);
    for (size_t j = 0; j < n; j++) {
        const double a = -2.0 * M_PI * (double)j / (double)n;
        h[j] = make_float2((float)cos(a), (float)sin(a));
    }
    for (size_t j = 0; j <= n; j++) {
        const double a = -2.0 * M_PI * (double)j / (double)(2 * n);
        h[n + j] = make_float2((float)cos(a), (float)sin(a));
    }
    float2 *d = nullptr;
    if (cudaMalloc(&d, sizeof(float2) * h.size()) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    // (pageable source: wait for the DMA itself, the Stockham kernels run on non-blocking streams -- see af_dev_upload)
    if (cudaMemcpy(d, h.data(), sizeof(float2) * h.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaStreamSynchronize(cudaStreamLegacy) != cudaSuccess) { cudaGetLastError(); cudaFree(d); return nullptr; }
    cache[dev][log2n] = d;
    return d;
}
