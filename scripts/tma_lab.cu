// Lab: how fast can one SM be FED with small source boxes?  Measures, per box shape, the rate at which
// per-warp rings of TMA tensor loads (mode 0), TMA loads + a 2 KB bulk copy (mode 1) or warp-issued
// 16-byte cp.async copies (mode 2) complete, with nothing consuming the data.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/tma_lab.bin scripts/tma_lab.cu
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}"
                 ::"r"(bar), "r"(parity) : "memory");
}

struct P {
    const unsigned char *src; const unsigned char *ent;
    int ps, np, bw, bh, depth, items, mode, stage_bytes, span;  // span: boxes are drawn from a window of `span` texel rows (L2 locality)
    unsigned long long *sink;
};

__global__ void __launch_bounds__(1024) lab(const __grid_constant__ CUtensorMap tm, const P p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    unsigned char *ring = smem + (size_t)warp * p.depth * p.stage_bytes;
    unsigned long long *bars = (unsigned long long *)(smem + (size_t)nw * p.depth * p.stage_bytes) + warp * p.depth;
    if (lane == 0)
        for (int s = 0; s < p.depth; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[s])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const int gw = blockIdx.x * nw + warp;
    unsigned rng = gw * 2654435761u + 12345u;
    const int box_bytes = p.bw * p.bh;
    auto issue = [&](int it) {
        const int s = it % p.depth;
        rng = rng * 1664525u + 1013904223u;
        const int x = ((rng >> 8) % (unsigned)(p.ps - p.bw)) & ~15;
        const int y = (rng >> 20) % (unsigned)(p.ps - p.bh);
        const int pl = (gw * 7 + it) % p.np;
        if (p.mode == 2) {
            const int cw = p.bw / 16, chunks = cw * p.bh;
            for (int c = lane; c < chunks; c += 32) {
                const int r = c / cw, cc = c - r * cw;
                const unsigned char *g = p.src + ((size_t)pl * p.ps + y + r) * p.ps + x + cc * 16;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(ring + s * p.stage_bytes + c * 16)), "l"(g) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            return;
        }
        if (lane == 0) {
            const unsigned bar = smem_u32(&bars[s]);
            const int extra = p.mode == 1 ? 2048 : 0;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(box_bytes + extra) : "memory");
            asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                         ::"r"(smem_u32(ring + s * p.stage_bytes)), "l"(&tm), "r"(x), "r"(y), "r"(pl), "r"(0), "r"(bar) : "memory");
            if (extra)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(ring + s * p.stage_bytes + box_bytes)), "l"(p.ent + (size_t)((gw * 131 + it * 7) & 8191) * 2048), "r"(extra), "r"(bar) : "memory");
        }
    };
    const int pre = p.depth < p.items ? p.depth : p.items;
    for (int it = 0; it < pre; ++it) issue(it);
    unsigned acc = 0;
    for (int it = 0; it < p.items; ++it) {
        const int s = it % p.depth;
        if (p.mode == 2) {
            asm volatile("cp.async.wait_group %0;" ::"n"(0) : "memory");  // depth-1 would need a constant; keep simple: drain
            __syncwarp();
        } else {
            mbar_wait(smem_u32(&bars[s]), (it / p.depth) & 1);
        }
        acc += ring[s * p.stage_bytes + lane * 4];
        __syncwarp();
        if (it + p.depth < p.items) issue(it + p.depth);
    }
    if (acc == 0x7fffffff) p.sink[0] = acc;
}

int main(int argc, char **argv) {
    const int ps = 2048, Pn = argc > 1 ? atoi(argv[1]) : 6;   // 6 plates = 25 MB (L2-resident), 96 = 403 MB (DRAM)
    const int promo = argc > 2 ? atoi(argv[2]) : 0;
    const int only_mode = argc > 3 ? atoi(argv[3]) : -1;
    unsigned char *d, *ent; unsigned long long *sink;
    cudaMalloc(&d, (size_t)ps * ps * Pn); cudaMemset(d, 1, (size_t)ps * ps * Pn);
    cudaMalloc(&ent, 8192 * 2048 + 4096); cudaMemset(ent, 2, 8192 * 2048 + 4096);
    cudaMalloc(&sink, 8);
    void *fn = nullptr; cudaDriverEntryPointQueryResult q;
    cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    const double ghz = prop.clockRate * 1e-6;
    printf("SMs %d clock %.3f GHz (nominal)\n", prop.multiProcessorCount, ghz);
    cudaFuncSetAttribute(lab, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    struct Shape { int bw, bh; } shapes[] = {{32, 32}, {48, 40}, {64, 32}, {64, 48}, {64, 64}, {128, 16}, {128, 32}, {256, 8}, {256, 16}, {96, 24}, {176, 16}, {16, 64}};
    printf("plates %d (%.0f MB) promotion %d\n", Pn, (double)ps * ps * Pn / 1e6, promo);
    for (int mode = 0; mode < 3; ++mode)
        for (auto sh : shapes)
            for (int warps_per_sm : {8, 16, 32}) {
                if (only_mode >= 0 && mode != only_mode) continue;
                const int depth = 2;
                P p; p.src = d; p.ent = ent; p.ps = ps; p.np = Pn; p.bw = sh.bw; p.bh = sh.bh; p.depth = depth; p.items = 400; p.mode = mode;
                p.stage_bytes = (sh.bw * sh.bh + (mode == 1 ? 2048 : 0) + 127) / 128 * 128; p.span = 0; p.sink = sink;
                CUtensorMap tm;
                cuuint64_t dims[4] = {(cuuint64_t)ps, (cuuint64_t)ps, (cuuint64_t)Pn, 1}, strides[3] = {(cuuint64_t)ps, (cuuint64_t)ps * ps, (cuuint64_t)ps * ps * Pn};
                cuuint32_t box[4] = {(cuuint32_t)sh.bw, (cuuint32_t)sh.bh, 1, 1}, es[4] = {1, 1, 1, 1};
                CUresult r = ((EncodeTiledFn)fn)(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                 CU_TENSOR_MAP_SWIZZLE_NONE, (CUtensorMapL2promotion)promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
                if (r != CUDA_SUCCESS) { printf("encode failed\n"); return 1; }
                // CTA = 8 warps; CTAs per SM = warps_per_sm / 8
                const int nw = 8, ctas = prop.multiProcessorCount * (warps_per_sm / nw);
                const size_t smem = (size_t)nw * depth * p.stage_bytes + nw * depth * 8;
                if (smem * (warps_per_sm / nw) > 220 * 1024) continue;
                cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
                lab<<<ctas, nw * 32, smem>>>(tm, p);
                cudaEventRecord(e0);
                lab<<<ctas, nw * 32, smem>>>(tm, p);
                cudaEventRecord(e1);
                cudaError_t e = cudaDeviceSynchronize();
                if (e != cudaSuccess) { printf("FAIL %s\n", cudaGetErrorString(e)); return 2; }
                float ms; cudaEventElapsedTime(&ms, e0, e1);
                const double boxes = (double)ctas * nw * p.items;
                const double bytes = boxes * (sh.bw * sh.bh + (mode == 1 ? 2048 : 0));
                printf("mode %d box %3dx%-3d warps/SM %2d: %.3f ms  %.1f Mbox/s/SM  %.1f GB/s total  %.1f B/clk/SM\n", mode, sh.bw, sh.bh, warps_per_sm, ms,
                       boxes / ms / 1e3 / prop.multiProcessorCount, bytes / ms / 1e6, bytes / (ms * 1e-3) / prop.multiProcessorCount / (1.9e9));
            }
    return 0;
}
