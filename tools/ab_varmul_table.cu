// ab_varmul_table.cu -- A/B of where k_varmul keeps its [P..8P] table (csrc/varmul.cuh): per-thread local memory (the
// library's choice) against thread-interleaved shared memory (entry k of thread t at s[k * blockDim + t], 160 doubles
// per thread).  Both kernels run varmul() on the same 2^20 random scalars times B and write the extended result;
// the outputs are compared and each kernel is timed with CUDA events (median of 21 launches after 3 warm-ups).
// Prints one JSON line.
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o ab_varmul_table tools/ab_varmul_table.cu
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../curve25519_dalek_b200/csrc/varmul.cuh"

struct SharedTab {
    double *base;
    __device__ double &at(int k) { return base[k * blockDim.x]; }
};

__device__ void load_pair(uint32_t s[8], ge64_p3 &P, const uint32_t *scalars, const uint64_t *pts, size_t i)
{
    for (int k = 0; k < 8; k++) s[k] = scalars[8 * i + k];
    s[7] &= 0x7fffffffu;
    ge_p3 p;
    fe_from_limbs51(p.X, pts + 20 * i); fe_from_limbs51(p.Y, pts + 20 * i + 5);
    fe_from_limbs51(p.Z, pts + 20 * i + 10); fe_from_limbs51(p.T, pts + 20 * i + 15);
    ge64_from_p3(P, p);
}

__device__ void store(double *out, const ge64_p3 &Q, size_t i)
{
    ge_p3 q; ge64_to_p3(q, Q);
    uint64_t l[20];
    fe_to_limbs51(l, q.X); fe_to_limbs51(l + 5, q.Y); fe_to_limbs51(l + 10, q.Z); fe_to_limbs51(l + 15, q.T);
    for (int k = 0; k < 20; k++) ((uint64_t *)out)[20 * i + k] = l[k];
}

__global__ void __launch_bounds__(128) k_local(const uint32_t *scalars, const uint64_t *pts, size_t n, double *out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8]; ge64_p3 P, Q;
    load_pair(s, P, scalars, pts, i);
    VarmulLocalTab tab;
    varmul(Q, s, P, tab);
    store(out, Q, i);
}

__global__ void __launch_bounds__(128) k_shared(const uint32_t *scalars, const uint64_t *pts, size_t n, double *out)
{
    extern __shared__ double s_tab[];
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8]; ge64_p3 P, Q;
    load_pair(s, P, scalars, pts, i);
    SharedTab tab{s_tab + threadIdx.x};
    varmul(Q, s, P, tab);
    store(out, Q, i);
}

template <class F>
static float median_ms(F launch)
{
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    for (int w = 0; w < 3; w++) launch();
    std::vector<float> t;
    for (int r = 0; r < 21; r++) {
        cudaEventRecord(a); launch(); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); t.push_back(ms);
    }
    std::sort(t.begin(), t.end());
    return t[t.size() / 2];
}

int main()
{
    const size_t n = (size_t)1 << 20;
    std::vector<uint32_t> hs(8 * n);
    uint64_t x = 0x9e3779b97f4a7c15ull;
    for (auto &w : hs) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; w = (uint32_t)x; }
    uint32_t *d_s; uint64_t *d_p; double *d_o1, *d_o2;
    cudaMalloc(&d_s, 32 * n); cudaMalloc(&d_p, 160 * n); cudaMalloc(&d_o1, 160 * n); cudaMalloc(&d_o2, 160 * n);
    cudaMemcpy(d_s, hs.data(), 32 * n, cudaMemcpyHostToDevice);
    // every point is B (extended limbs); the multiplication's cost does not depend on the point
    ge_p3 B; ge_p3_basepoint(B);
    uint64_t lb[20];
    fe_to_limbs51(lb, B.X); fe_to_limbs51(lb + 5, B.Y); fe_to_limbs51(lb + 10, B.Z); fe_to_limbs51(lb + 15, B.T);
    std::vector<uint64_t> hp(20 * n);
    for (size_t i = 0; i < n; i++) memcpy(&hp[20 * i], lb, 160);
    cudaMemcpy(d_p, hp.data(), 160 * n, cudaMemcpyHostToDevice);
    const unsigned blocks = (unsigned)((n + 127) / 128);
    const int smem = 128 * 8 * VARMUL_ENTRY * sizeof(double);
    cudaFuncSetAttribute(k_shared, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    const float t_local = median_ms([&] { k_local<<<blocks, 128>>>(d_s, d_p, n, d_o1); });
    const float t_shared = median_ms([&] { k_shared<<<blocks, 128, smem>>>(d_s, d_p, n, d_o2); });
    std::vector<uint64_t> o1(20 * n), o2(20 * n);
    cudaMemcpy(o1.data(), d_o1, 160 * n, cudaMemcpyDeviceToHost);
    cudaMemcpy(o2.data(), d_o2, 160 * n, cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    printf("{\"n\": %zu, \"local_ms\": %.3f, \"local_per_s\": %.0f, \"shared_ms\": %.3f, \"shared_per_s\": %.0f, "
           "\"shared_bytes_per_block\": %d, \"outputs_equal\": %s, \"cuda\": \"%s\"}\n",
           n, t_local, n / t_local * 1e3, t_shared, n / t_shared * 1e3, smem, o1 == o2 ? "true" : "false", cudaGetErrorString(e));
    return e == cudaSuccess && o1 == o2 ? 0 : 1;
}
