// fused_ceiling — measurement tool (not product): what can k_fused's data movement reach on this GPU?
// The bench's layout: 64 runs x 4 MiB = 256 MiB of input in 8 KiB tiles, every tile loaded into shared memory with one TMA bulk load and
// stored back with one TMA bulk store to the same offsets of a second 256 MiB buffer.  Reported as TB/s of read + write bytes for
//   copy     cudaMemcpyAsync device to device (the practical copy ceiling)
//   perwarp  the skeleton of k_fused: one CTA per SM, 16 or 12 warps, one 10 KB buffer per warp; wait for the previous store to drain,
//            load, (L2 prefetch of the warp's next tile), wait, store
//   ring     one CTA per SM, one producer warp filling a ring of S stages (full / empty mbarriers) for N consumer warps; a consumer
//            releases a stage once its store has been read, either at once (defer 0) or after its next item's store was issued
//            (defer 1).  The shape DESIGN §9.1 measured and did not take
// `spin` is a stand-in for the decode: every tile holds its warp that many SM cycles between load and store.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/probes/fused_ceiling tools/probes/fused_ceiling.cu
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>
#include <algorithm>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

constexpr uint32_t kTile = 8192, kBuf = 10240;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* s, const void* g, uint32_t n, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(s)), "l"(g), "r"(n), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* g, const void* s, uint32_t n) { asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"(smem_u32(s)), "r"(n) : "memory"); }
__device__ __forceinline__ void bulk_prefetch_l2(const void* g, uint32_t n) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(g), "r"(n) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void spin(uint32_t cycles) { if (cycles) { const long long t0 = clock64(); while (clock64() - t0 < cycles) {} } }

struct PerWarpSmem { alignas(128) uint8_t buf[kBuf]; alignas(8) unsigned long long mbar; };
__global__ void k_perwarp(const uint8_t* src, uint8_t* dst, uint32_t n_tiles, uint32_t warps, int prefetch, uint32_t spin_cycles) {
    extern __shared__ __align__(128) uint8_t raw[];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    PerWarpSmem& S = reinterpret_cast<PerWarpSmem*>(raw)[wid];
    if (lane == 0) { mbar_init(&S.mbar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncwarp();
    uint32_t phase = 0;
    const uint32_t n_warps = gridDim.x * warps;
    for (uint32_t t = blockIdx.x * warps + wid; t < n_tiles; t += n_warps) {
        if (lane == 0) {
            bulk_wait_read<0>(); mbar_arrive_expect_tx(&S.mbar, kTile); bulk_g2s(S.buf, src + (size_t)t * kTile, kTile, &S.mbar);
            if (prefetch && t + n_warps < n_tiles) bulk_prefetch_l2(src + (size_t)(t + n_warps) * kTile, kTile);
        }
        __syncwarp();
        mbar_wait(&S.mbar, phase & 1u); phase++;
        spin(spin_cycles);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) { bulk_s2g(dst + (size_t)t * kTile, S.buf, kTile); bulk_commit(); }
        __syncwarp();
    }
    if (lane == 0) bulk_wait<0>();
}

struct alignas(128) RingStage { uint8_t buf[kBuf]; uint32_t tile, seq; };
struct RingBars { unsigned long long full, empty; };
// dynamic smem: S stages, then S barrier pairs
// defer 1: after storing item k, wait for all but that store to be read and release item k-1; defer 0: wait for item k's store to be read
// and release item k at once
__global__ void k_ring(const uint8_t* src, uint8_t* dst, uint32_t n_tiles, uint32_t S, uint32_t spin_cycles, int defer) {
    extern __shared__ __align__(128) uint8_t raw[];
    RingStage* st = reinterpret_cast<RingStage*>(raw);
    RingBars* bars = reinterpret_cast<RingBars*>(raw + S * sizeof(RingStage));
    __shared__ uint32_t s_ticket;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, n_cons = blockDim.x / 32 - 1;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < S; s++) { mbar_init(&bars[s].full, 1); mbar_init(&bars[s].empty, 1); st[s].seq = ~0u; }
        s_ticket = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (wid == 0) {
        if (lane == 0) {
            const uint32_t t0 = (uint32_t)((uint64_t)n_tiles * blockIdx.x / gridDim.x), t1 = (uint32_t)((uint64_t)n_tiles * (blockIdx.x + 1) / gridDim.x);
            uint32_t k = 0;
            for (uint32_t t = t0; t < t1 + n_cons; t++, k++) {
                const uint32_t s = k % S;
                mbar_wait(&bars[s].empty, ((k / S) & 1u) ^ 1u);
                *(volatile uint32_t*)&st[s].seq = k;
                if (t < t1) {
                    st[s].tile = t;
                    mbar_arrive_expect_tx(&bars[s].full, kTile); bulk_g2s(st[s].buf, src + (size_t)t * kTile, kTile, &bars[s].full);
                } else { st[s].tile = ~0u; mbar_arrive(&bars[s].full); }
            }
        }
        return;
    }
    uint32_t prev = ~0u;
    for (;;) {
        uint32_t k = 0;
        if (lane == 0) k = atomicAdd(&s_ticket, 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (prev != ~0u && k - prev >= S) {               // the producer needs prev's stage before it can fill k's: release it now
            if (lane == 0) { bulk_wait_read<0>(); mbar_arrive(&bars[prev % S].empty); }
            prev = ~0u;
        }
        const uint32_t s = k % S;
        // a ticket can run more than S items ahead of the stage's last consumer, and a parity wait cannot tell phases two apart: wait
        // until the producer has taken the stage for item k (so the stage's full barrier is in k's phase), then for the phase
        while (*(volatile uint32_t*)&st[s].seq != k) {}
        mbar_wait(&bars[s].full, (k / S) & 1u);
        const uint32_t t = st[s].tile;
        if (t == ~0u) { if (lane == 0) mbar_arrive(&bars[s].empty); break; }
        spin(spin_cycles);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
            bulk_s2g(dst + (size_t)t * kTile, st[s].buf, kTile); bulk_commit();
            if (defer) { bulk_wait_read<1>(); if (prev != ~0u) mbar_arrive(&bars[prev % S].empty); }
            else { bulk_wait_read<0>(); mbar_arrive(&bars[s].empty); }
        }
        __syncwarp();
        prev = defer ? k : ~0u;
    }
    if (lane == 0) { bulk_wait<0>(); if (prev != ~0u) mbar_arrive(&bars[prev % S].empty); }
}

static double median(std::vector<double> v) { std::sort(v.begin(), v.end()); return v[v.size() / 2]; }

int main(int argc, char** argv) {
    const size_t N = 256ull << 20;
    const uint32_t n_tiles = (uint32_t)(N / kTile);
    const int reps = argc > 1 ? atoi(argv[1]) : 7;
    uint8_t *src, *dst; CK(cudaMalloc(&src, N)); CK(cudaMalloc(&dst, N));
    CK(cudaMemset(src, 0x5a, N)); CK(cudaMemset(dst, 0, N));
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    int clk_khz = 0; CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s, %d SMs, L2 %d MB, max SM clock %d MHz\n", prop.name, sms, prop.l2CacheSize >> 20, clk_khz / 1000);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int inner = 10;
    // read + write bytes per pass, over the median of `reps` timings of `inner` passes; min and max give the spread
    std::vector<uint8_t> h(N);
    size_t bad = 0;
    auto report = [&](const char* what, auto&& launch) {
        CK(cudaMemset(dst, 0, N));
        launch(); CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), dst, N, cudaMemcpyDeviceToHost));             // the skeleton moved every byte
        for (size_t i = 0; i < N; i++) bad += h[i] != 0x5a;
        std::vector<double> tb;
        for (int r = 0; r < reps; r++) {
            cudaEventRecord(e0);
            for (int i = 0; i < inner; i++) launch();
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            tb.push_back(2.0 * N * inner / (ms * 1e-3) / 1e12);
        }
        const double med = median(tb);
        printf("%-40s %7.1f us/pass  %.3f TB/s  (min %.3f max %.3f)\n", what, 2.0 * N / (med * 1e12) * 1e6, med, *std::min_element(tb.begin(), tb.end()), *std::max_element(tb.begin(), tb.end()));
    };
    report("copy cudaMemcpyAsync D2D", [&] { CK(cudaMemcpyAsync(dst, src, N, cudaMemcpyDeviceToDevice)); });
    const uint32_t spins[] = { 0, 2000, 4000, 8000 };
    for (uint32_t sp : spins) {
        for (uint32_t warps : { 16u, 12u }) {
            const size_t smem = sizeof(PerWarpSmem) * warps;
            CK(cudaFuncSetAttribute(k_perwarp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            for (int pf = 1; pf >= 0; pf--) {
                char name[96]; snprintf(name, sizeof name, "perwarp w%u prefetch %d spin %u", warps, pf, sp);
                report(name, [&] { k_perwarp<<<sms, warps * 32, smem>>>(src, dst, n_tiles, warps, pf, sp); });
            }
        }
        const uint32_t cfg[][2] = { { 8, 7 }, { 16, 7 }, { 16, 11 }, { 20, 11 }, { 20, 15 } };
        for (auto& c : cfg) {
            const uint32_t S = c[0], n_cons = c[1];
            const size_t smem = S * (sizeof(RingStage) + sizeof(RingBars));
            CK(cudaFuncSetAttribute(k_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            for (int defer = 1; defer >= 0; defer--) {
                char name[96]; snprintf(name, sizeof name, "ring S %u consumers %u defer %d spin %u", S, n_cons, defer, sp);
                report(name, [&] { k_ring<<<sms, (n_cons + 1) * 32, smem>>>(src, dst, n_tiles, S, sp, defer); });
            }
        }
    }
    printf("dst check: %zu wrong bytes\n", bad);
    return bad != 0;
}
