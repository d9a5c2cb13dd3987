// l2_probe.cu -- L2 throughput of layouts of the f-k column passes' level-A/B intermediate V.
//
// V is a ring of 5 chunks x 13 planes x 400 rows x 80 sample pairs x 16 B (33 MB, the ring of the 10 000-channel
// plan), kept in L2 with the evict_last policy the column kernels use.  Position of pair p inside a row, per layout:
//   natural: p                                       (the order before: level A's accesses are half sectors)
//   split:   (p >> 1) + (p & 1) * 40                 (even pairs in the first half of the row, odd in the second)
//   blocked: (p & ~7) | ((p >> 1) & 3) | ((p & 1) << 2)   (the same inside each 8-pair, 128-byte group)
// Two access shapes, as in the kernels:
//   A: a thread owns a quad (pairs 2q, 2q + 1 of a row), consecutive threads consecutive quads: two 16-byte accesses
//   B: a thread owns one pair of an 8-pair tile, a warp the same tile of 4 rows: one 16-byte access
// Each test runs REPS passes over the ring per launch and is timed with CUDA events:
//   store : st.global.L2::cache_hint (evict_last);  load : ld.global.cg.L2::cache_hint (evict_last)
//   mixed : shape A, like one column pass: two 16-byte loads of x streamed from HBM (evict_first), two V stores, two V
//           loads from the ring slot two chunks behind
// Output: one line per test with the time per launch, the useful bytes per second and the L2 sector bytes per second
// (shape A in the natural layout moves two sectors for every sector of data).
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o l2_probe scripts/l2_probe.cu && ./l2_probe
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } \
    } while (0)

constexpr unsigned kPairs = 80, kH = kPairs / 2;                 // sample pairs per chunk row, half of it
constexpr unsigned kRows = 5u * 13u * 400u;                      // ring slots x planes x c2 rows
constexpr unsigned kQuads = kRows * kH;                          // quads in the ring
constexpr unsigned kSlotQuads = kQuads / 5;
constexpr unsigned kReps = 20;                                   // ring passes per launch
constexpr size_t kXElems = (size_t)1 << 27;                      // 2 GiB of x, far larger than L2

__device__ __forceinline__ unsigned long long pol_last() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ unsigned long long pol_first() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ float4 ld16(const float4* p, unsigned long long pol) {
    float4 r;
    asm volatile("ld.global.cg.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol) : "memory");
    return r;
}
__device__ __forceinline__ void st16(float4* p, float4 v, unsigned long long pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

enum { NATURAL = 0, SPLIT = 1, BLOCKED = 2 };
static const char* kLayoutName[] = {"natural", "split", "blocked"};

template <int LAYOUT>
__device__ __forceinline__ unsigned pos(unsigned p) {
    if (LAYOUT == NATURAL) return p;
    if (LAYOUT == SPLIT) return (p >> 1) + (p & 1) * kH;
    return (p & ~7u) | ((p >> 1) & 3u) | ((p & 1u) << 2);
}

// shape A: element offsets of quad q's two pairs in the ring
template <int LAYOUT>
__device__ __forceinline__ void quad_pos(unsigned q, unsigned& a, unsigned& b) {
    const unsigned row = q / kH, t4 = q - row * kH;
    a = row * kPairs + pos<LAYOUT>(2 * t4);
    b = row * kPairs + pos<LAYOUT>(2 * t4 + 1);
}

enum { STORE_A = 0, LOAD_A = 1, STORE_B = 2, LOAD_B = 3, MIXED = 4 };
static const char* kModeName[] = {"store A", "load A", "store B", "load B", "mixed x+st+ld A"};

template <int MODE, int LAYOUT>
__global__ void __launch_bounds__(256) k_probe(float4* ring, const float4* __restrict__ x, float4* sink) {
    const unsigned long long keep = pol_last(), stream = pol_first();
    const unsigned stride = gridDim.x * blockDim.x;
    const bool shape_b = MODE == STORE_B || MODE == LOAD_B;
    const unsigned n = kReps * (shape_b ? 2 * kQuads : kQuads);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < n; g += stride) {
        if (shape_b) {
            // as level B's items (c2 row n, pair j): a warp is 4 rows x the same 8-pair tile
            const unsigned e = g % (2 * kQuads), j = e & 7u, r4 = (e >> 3) & 3u, t = e >> 5;
            const unsigned row = (t / (kPairs / 8)) * 4 + r4, p = (t % (kPairs / 8)) * 8 + j;
            float4* a = ring + row * kPairs + pos<LAYOUT>(p);
            if (MODE == STORE_B) {
                st16(a, make_float4((float)g, 0.f, 0.f, 0.f), keep);
            } else {
                const float4 u = ld16(a, keep);
                acc.x += u.x; acc.y += u.y; acc.z += u.z; acc.w += u.w;
            }
            continue;
        }
        const unsigned q = g % kQuads;
        unsigned a, b;
        quad_pos<LAYOUT>(q, a, b);
        if (MODE == STORE_A) {
            const float4 v = make_float4((float)g, 0.f, 0.f, 0.f);
            st16(ring + a, v, keep); st16(ring + b, v, keep);
        } else if (MODE == LOAD_A) {
            const float4 u = ld16(ring + a, keep), v = ld16(ring + b, keep);
            acc.x += u.x + v.x; acc.y += u.y + v.y; acc.z += u.z + v.z; acc.w += u.w + v.w;
        } else {
            const float4* xs = x + (2 * (size_t)g) % kXElems;
            const float4 u = ld16(xs, stream), v = ld16(xs + 1, stream);
            st16(ring + a, u, keep); st16(ring + b, v, keep);
            unsigned ra, rb;
            quad_pos<LAYOUT>((q + 2 * kSlotQuads) % kQuads, ra, rb);
            const float4 s = ld16(ring + ra, keep), t = ld16(ring + rb, keep);
            acc.x += s.x + t.x; acc.y += s.y + t.y; acc.z += s.z + t.z; acc.w += s.w + t.w;
        }
    }
    if (acc.x == 1.2345e-30f) sink[0] = acc;           // never true for these data; keeps the sums live
}

template <int MODE, int LAYOUT>
static void run(float4* ring, const float4* x, float4* sink, int grid) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) k_probe<MODE, LAYOUT><<<grid, 256>>>(ring, x, sink);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<float> ms;
    for (int i = 0; i < 15; ++i) {
        CK(cudaEventRecord(e0));
        k_probe<MODE, LAYOUT><<<grid, 256>>>(ring, x, sink);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float t; CK(cudaEventElapsedTime(&t, e0, e1));
        ms.push_back(t);
    }
    std::sort(ms.begin(), ms.end());
    const double med = ms[ms.size() / 2];
    // V bytes per pass over the ring, 32 B per quad; the mixed test stores and loads V and reads as many bytes of x
    const double v = (double)kReps * kQuads * 32.0;
    const double v_kinds = MODE == MIXED ? 2.0 : 1.0;
    const bool half = LAYOUT == NATURAL && MODE != STORE_B && MODE != LOAD_B;   // shape A, natural order: half sectors
    const double useful = v * v_kinds + (MODE == MIXED ? v : 0.0);
    const double sectors = v * v_kinds * (half ? 2.0 : 1.0) + (MODE == MIXED ? v : 0.0);
    printf("%-16s %-8s  %8.3f ms  (min %8.3f, max %8.3f)  useful %7.1f GB/s  L2 sectors %7.1f GB/s\n", kModeName[MODE],
           kLayoutName[LAYOUT], med, ms.front(), ms.back(), useful / med * 1e-6, sectors / med * 1e-6);
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
}

template <int MODE>
static void run_layouts(float4* ring, const float4* x, float4* sink, int grid) {
    run<MODE, NATURAL>(ring, x, sink, grid);
    run<MODE, SPLIT>(ring, x, sink, grid);
    run<MODE, BLOCKED>(ring, x, sink, grid);
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s, %d SMs, L2 %d MB; ring %.2f MB (%u quads), %u passes per launch\n", prop.name,
           prop.multiProcessorCount, prop.l2CacheSize >> 20, kQuads * 32.0 / 1e6, kQuads, kReps);
    float4 *ring, *x, *sink;
    CK(cudaMalloc(&ring, (size_t)kQuads * 32));
    CK(cudaMalloc(&x, kXElems * 16));
    CK(cudaMalloc(&sink, 16));
    CK(cudaMemset(ring, 0, (size_t)kQuads * 32));
    CK(cudaMemset(x, 0, kXElems * 16));
    const int grid = prop.multiProcessorCount * 8;
    // the layouts run back to back, twice, so that drifting clocks touch all of them
    for (int round = 0; round < 2; ++round) {
        printf("-- round %d\n", round);
        run_layouts<STORE_A>(ring, x, sink, grid);
        run_layouts<LOAD_A>(ring, x, sink, grid);
        run_layouts<STORE_B>(ring, x, sink, grid);
        run_layouts<LOAD_B>(ring, x, sink, grid);
        run_layouts<MIXED>(ring, x, sink, grid);
    }
    CK(cudaFree(ring)); CK(cudaFree(x)); CK(cudaFree(sink));
    return 0;
}
