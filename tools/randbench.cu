// Microbenchmark: how many independent random 32-byte sector reads per second does the GPU sustain
// over a table of a given size?  This is the hardware ceiling for the k-mer table probes of
// match_kernel (one random sector per probe, no reuse), as opposed to the streaming-copy bandwidth
// in MEASURED_PEAKS.json.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/randbench tools/randbench.cu
//   tools/randbench [table_GiB ...]          (RB_FULL=1: also dependent chains, 32-byte L2 fetch granularity,
//                                             64/128-byte accesses; RB_VMM=1: table mapped with cuMemCreate/cuMemMap)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda.h>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDULL; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ULL; x ^= x >> 33;
  return x;
}
__device__ __forceinline__ void ld256(const void* p, uint32_t (&w)[8]) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}

// MLP independent loads in flight per thread, `iters` rounds; dependent = 1 chains the next address on the data
// Same, but every access reads W consecutive sectors of one W*32-byte aligned line (bucketised tables)
template <int W>
__global__ void __launch_bounds__(256) wide_kernel(const uint8_t* tab, uint64_t mask, int iters, uint32_t* sink) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t s = mix64(tid + 1);
  uint32_t acc = 0;
  for (int i = 0; i < iters; ++i) {
    uint32_t v[W][8];
    const uint8_t* a = tab + (((s & mask) & ~(uint64_t)(W - 1)) << 5);
#pragma unroll
    for (int j = 0; j < W; ++j) ld256(a + 32 * j, v[j]);
#pragma unroll
    for (int j = 0; j < W; ++j) acc ^= v[j][0] ^ v[j][7];
    s = mix64(s + v[0][3] + 0x9E3779B97F4A7C15ULL);
  }
  if (acc == 0x12345678u) sink[0] = acc;
}

template <int MLP>
__global__ void __launch_bounds__(256) probe_kernel(const uint8_t* tab, uint64_t mask, int iters, int dependent, uint32_t* sink) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t s[MLP];
  for (int j = 0; j < MLP; ++j) s[j] = mix64(tid * MLP + j + 1);
  uint32_t acc = 0;
  for (int i = 0; i < iters; ++i) {
    uint32_t v[MLP][8];
#pragma unroll
    for (int j = 0; j < MLP; ++j) ld256(tab + ((s[j] & mask) << 5), v[j]);
#pragma unroll
    for (int j = 0; j < MLP; ++j) {
      acc ^= v[j][0] ^ v[j][7];
      s[j] = mix64(s[j] + (dependent ? v[j][3] : 0u) + 0x9E3779B97F4A7C15ULL);
    }
  }
  if (acc == 0x12345678u) sink[0] = acc;
}

// Table through the virtual-memory API (cuMemCreate + cuMemMap): lets the driver pick its largest page size
static uint8_t* vmm_alloc(size_t bytes, size_t align, size_t* gran_out) {
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = 0;
  size_t gmin = 0, grec = 0;
  cuMemGetAllocationGranularity(&gmin, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
  cuMemGetAllocationGranularity(&grec, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
  fprintf(stderr, "vmm granularity: minimum %zu recommended %zu\n", gmin, grec);
  *gran_out = grec;
  const size_t sz = (bytes + align - 1) / align * align;
  CUdeviceptr va = 0;
  if (cuMemAddressReserve(&va, sz, align, 0, 0) != CUDA_SUCCESS) return nullptr;
  CUmemGenericAllocationHandle h;
  if (cuMemCreate(&h, sz, &prop, 0) != CUDA_SUCCESS) return nullptr;
  if (cuMemMap(va, sz, 0, h, 0) != CUDA_SUCCESS) return nullptr;
  CUmemAccessDesc acc = {};
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (cuMemSetAccess(va, sz, &acc, 1) != CUDA_SUCCESS) return nullptr;
  return (uint8_t*)va;
}

int main(int argc, char** argv) {
  std::vector<double> sizes;
  for (int i = 1; i < argc; ++i) sizes.push_back(atof(argv[i]));
  if (sizes.empty()) sizes = {0.0625, 1, 4, 16};
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  uint32_t* sink;
  cudaMalloc(&sink, 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const bool use_vmm = getenv("RB_VMM") != nullptr;
  const bool full = getenv("RB_FULL") != nullptr;      // default: one line per table size (what bench.py reads)
  cudaFree(0);
  for (int gran : {0, 32}) {
    if (gran && !full) break;
    if (gran) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
    size_t g = 0;
    cudaDeviceGetLimit(&g, cudaLimitMaxL2FetchGranularity);
    for (double gib : sizes) {
      uint64_t slots = 1;
      while ((double)(slots * 2) * 32 <= gib * 1073741824.0) slots *= 2;
      uint8_t* tab = nullptr;
      size_t vg = 0;
      if (use_vmm) {
        tab = vmm_alloc(slots * 32, (size_t)512 << 20, &vg);
        if (!tab) { printf("vmm alloc %.2f GiB failed\n", gib); continue; }
      } else if (cudaMalloc(&tab, slots * 32) != cudaSuccess) { printf("alloc %.2f GiB failed\n", gib); cudaGetLastError(); continue; }
      cudaMemset(tab, 1, slots * 32);
      for (int dep = 0; dep < (full ? 2 : 1); ++dep)
        for (int tpsm : {1536}) {
          const int blocks = sms * tpsm / 256, iters = 64;
          auto run = [&](int mlp) {
            if (mlp == 1) probe_kernel<1><<<blocks, 256>>>(tab, slots - 1, iters, dep, sink);
            else if (mlp == 2) probe_kernel<2><<<blocks, 256>>>(tab, slots - 1, iters, dep, sink);
            else probe_kernel<4><<<blocks, 256>>>(tab, slots - 1, iters, dep, sink);
          };
          for (int mlp : {4}) {
            run(mlp);
            cudaDeviceSynchronize();
            cudaEventRecord(e0);
            for (int r = 0; r < 3; ++r) run(mlp);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            const double n = 3.0 * blocks * 256.0 * iters * mlp;
            printf("{\"l2_fetch_gran\": %zu, \"table_gib\": %.4f, \"dependent\": %d, \"threads_per_sm\": %d, \"mlp\": %d, \"gsectors_per_s\": %.2f, \"gb_per_s_32B\": %.1f}\n",
                   g, slots * 32 / 1073741824.0, dep, tpsm, mlp, n / ms / 1e6, n * 32 / ms / 1e6);
            fflush(stdout);
          }
        }
      for (int w : {1, 2, 4}) {
        if (!full) break;
        const int blocks = sms * 1536 / 256, iters = 64;
        auto run = [&]() {
          if (w == 1) wide_kernel<1><<<blocks, 256>>>(tab, slots - 1, iters, sink);
          else if (w == 2) wide_kernel<2><<<blocks, 256>>>(tab, slots - 1, iters, sink);
          else wide_kernel<4><<<blocks, 256>>>(tab, slots - 1, iters, sink);
        };
        run();
        cudaDeviceSynchronize();
        cudaEventRecord(e0);
        for (int r = 0; r < 3; ++r) run();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        const double n = 3.0 * blocks * 256.0 * iters;
        printf("{\"l2_fetch_gran\": %zu, \"table_gib\": %.4f, \"access_bytes\": %d, \"threads_per_sm\": 1536, \"gaccesses_per_s\": %.2f}\n",
               g, slots * 32 / 1073741824.0, 32 * w, n / ms / 1e6);
        fflush(stdout);
      }
      if (!use_vmm) cudaFree(tab);
    }
  }
  return 0;
}
