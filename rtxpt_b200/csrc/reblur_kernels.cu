// reblur_kernels.cu — NRD's REBLUR_DIFFUSE_SPECULAR chain for one stable plane (SURVEY §8 row a18 / K9), one kernel per pass of the dispatch graph the settings select
// (the pass bodies live in reblur_passes.cuh; see there for the per-pass citations).  One thread per pixel, 16x16 CTAs aligned to NRD's 16x16 sky tiles, taps fetched through L2
// (the working set of one plane at 1080p is ~90 MB, larger than the 50 MB L2, so a pass streams its inputs while its taps hit L1 / L2).  The passes are ALU-heavy (thousands
// of thread-instructions per pixel per pass, a few hundred bytes) - so tiling pays through the arithmetic it removes (per-tap unpacking, clamped addressing), not through bandwidth: the 5x5 / 3x3 pass stages its
// neighbourhood with TMA (below); the Poisson-tap passes reach up to 40 pixels away and keep reading through L1 / L2.
#include "reblur_passes.cuh"
#include "reblur_host.h"
#include "kernels.h"
#include <cstdlib>
#include <cstring>
#include <cuda.h>            // CUtensorMap (the encoder is fetched through cudaGetDriverEntryPoint: no link dependency on libcuda)

namespace pt { namespace rb {

#define RB_XY const int x = int(blockIdx.x * 16 + threadIdx.x), y = int(blockIdx.y * 16 + threadIdx.y); if (x >= int(p.W) || y >= int(p.H)) return

__global__ void __launch_bounds__(256) k_rb_classify_tiles(const __grid_constant__ Params p)
{
    const int sky = __syncthreads_count(beyondDenoisingRange(p, int(blockIdx.x * 16 + threadIdx.x), int(blockIdx.y * 16 + threadIdx.y)));
    if (threadIdx.x == 0 && threadIdx.y == 0) p.tiles[blockIdx.y * p.tilesW + blockIdx.x] = sky == 256 ? 1 : 0;
}
template <int RADIUS> __global__ void __launch_bounds__(256) k_rb_hit_dist_reconstruction(const __grid_constant__ Params p) { RB_XY; hitDistReconstructionPixel<RADIUS>(p, x, y); }

// ---- tiled HitDistReconstruction: the neighbourhood of a 16x16 tile (24 x 20 texels for the 5x5 taps, 24 x 18 for the 3x3 ones, see below) staged in shared memory by four 2-D TMA tensor loads ------
// (viewZ R32F, normal/roughness R10G10B10A2 as u32, diffuse and specular radiance + hit distance RGBA16F as u64), one mbarrier, the normals unpacked once per texel instead of
// once per tap.  TMA fills out-of-image texels with zeros where the pass wants clamped coordinates, so the tiles on the image border - and images whose row pitch is not a
// multiple of 16 bytes, which TMA cannot address - load their region with ordinary clamped loads; both ways the shared tile holds the same values.
// TMA wants the byte offset of a box's first texel in a row to be a multiple of 16 (measured: a box starting at x = 30 of a 32-bit image raises "illegal instruction", x = 32 loads -
// scripts/probes/tma_probe2.cu), so the region starts 4 texels left of the tile (16 B for the 32-bit images, 32 B for the 64-bit ones) and is 24 wide (a box row must also be a
// multiple of 16 B): columns 2..21 are the 5x5 taps' reach, 3..20 the 3x3 taps'.  Rows: the tile and RADIUS rows above and below it, the rows the taps read.
constexpr int kHdTile = 16, kHdLeft = 4, kHdRegionW = kHdTile + kHdLeft + 4;
template <int RADIUS> struct HitDistRegion
{
    static constexpr int H = kHdTile + 2 * RADIUS, texels = kHdRegionW * H;
    static constexpr int stride = (texels + 31) / 32 * 32;             // array length: every array of the tile starts on a 128-byte boundary (TMA destination alignment)
};
struct HitDistTileMaps { CUtensorMap viewZ, normalRoughness, diff, spec; uint useTma; };
template <int RADIUS> struct __align__(128) HitDistTile
{
    static constexpr int kTexels = HitDistRegion<RADIUS>::stride;
    float viewZ[kTexels];                           // 5x5: 1920 B each for the 32-bit images, 3840 B for the 64-bit ones
    uint normalRoughness[kTexels];
    unsigned long long diff[kTexels];
    unsigned long long spec[kTexels];
    float4 unpacked[kTexels];                       // normal.xyz, roughness
    unsigned long long mbar;
};
static_assert(offsetof(HitDistTile<2>, normalRoughness) % 128 == 0 && offsetof(HitDistTile<2>, diff) % 128 == 0 && offsetof(HitDistTile<2>, spec) % 128 == 0, "TMA destinations must be 128-byte aligned");
static_assert(offsetof(HitDistTile<1>, normalRoughness) % 128 == 0 && offsetof(HitDistTile<1>, diff) % 128 == 0 && offsetof(HitDistTile<1>, spec) % 128 == 0, "TMA destinations must be 128-byte aligned");
template <int RADIUS> struct SharedTaps
{
    const Params& p; const HitDistTile<RADIUS>& t; int x0, y0;  // texel (x0, y0) of the image is cell 0 of the region
    __device__ int cell(int qx, int qy) const { return (qy - y0) * kHdRegionW + (qx - x0); }
    __device__ float viewZ(int qx, int qy) const { return fabsf(t.viewZ[cell(qx, qy)] * p.viewZScale); }
    __device__ float4 normalRoughness(int qx, int qy) const { return t.unpacked[cell(qx, qy)]; }
    __device__ float diffHitDist(int qx, int qy) const { return f16tof32(uint(t.diff[cell(qx, qy)] >> 48)); }
    __device__ float specHitDist(int qx, int qy) const { return f16tof32(uint(t.spec[cell(qx, qy)] >> 48)); }
};
__device__ __forceinline__ void tmaLoadTile2D(void* smemDst, const CUtensorMap* map, int x, int y, unsigned long long* mbar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"((uint)__cvta_generic_to_shared(smemDst)), "l"(map), "r"(x), "r"(y), "r"((uint)__cvta_generic_to_shared(mbar)) : "memory");
}
template <int RADIUS> __global__ void __launch_bounds__(256) k_rb_hit_dist_reconstruction_tiled(const __grid_constant__ Params p, const __grid_constant__ HitDistTileMaps maps)
{
    constexpr int kHdRegionH = HitDistRegion<RADIUS>::H, kHdTexels = HitDistRegion<RADIUS>::texels;
    __shared__ HitDistTile<RADIUS> tile;
    if (p.tiles[blockIdx.y * p.tilesW + blockIdx.x]) return;                        // sky tile: nothing to reconstruct (uniform over the CTA)
    const int tid = int(threadIdx.y * 16 + threadIdx.x), W = int(p.W), H = int(p.H);
    const int x0 = int(blockIdx.x) * kHdTile - kHdLeft, y0 = int(blockIdx.y) * kHdTile - RADIUS;
    const bool interior = x0 >= 0 && y0 >= 0 && x0 + kHdRegionW <= W && y0 + kHdRegionH <= H;
    if (maps.useTma && interior)
    {
        const uint mbarAddr = (uint)__cvta_generic_to_shared(&tile.mbar);
        if (tid == 0)
        {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbarAddr));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbarAddr), "r"(uint(kHdTexels * (4 + 4 + 8 + 8))) : "memory");
            tmaLoadTile2D(tile.viewZ, &maps.viewZ, x0, y0, &tile.mbar);
            tmaLoadTile2D(tile.normalRoughness, &maps.normalRoughness, x0, y0, &tile.mbar);
            tmaLoadTile2D(tile.diff, &maps.diff, x0, y0, &tile.mbar);
            tmaLoadTile2D(tile.spec, &maps.spec, x0, y0, &tile.mbar);
        }
        __syncthreads();                                                            // the barrier is initialised before anyone polls it
        uint done = 0;
        while (!done) asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0; selp.u32 %0, 1, 0, q; }" : "=r"(done) : "r"(mbarAddr) : "memory");
    }
    else
    {
        for (int c = tid; c < kHdTexels; c += 256)
        {
            const int qx = clampi(x0 + c % kHdRegionW, 0, W - 1), qy = clampi(y0 + c / kHdRegionW, 0, H - 1); const size_t q = size_t(qy) * W + qx;
            tile.viewZ[c] = p.viewZ[q]; tile.normalRoughness[c] = p.normalRoughness[q];
            const uint2 d = p.inDiff[q], s = p.inSpec[q];
            tile.diff[c] = (unsigned long long)d.x | ((unsigned long long)d.y << 32); tile.spec[c] = (unsigned long long)s.x | ((unsigned long long)s.y << 32);
        }
        __syncthreads();
    }
    for (int c = tid; c < kHdTexels; c += 256) { float m; tile.unpacked[c] = unpackNormalRoughness(tile.normalRoughness[c], m); }
    __syncthreads();
    const int x = int(blockIdx.x * 16 + threadIdx.x), y = int(blockIdx.y * 16 + threadIdx.y);
    if (x >= W || y >= H) return;
    const SharedTaps<RADIUS> taps{ p, tile, x0, y0 };
    hitDistReconstructionBody<RADIUS>(p, x, y, taps);
}
template <int MODE> __global__ void __launch_bounds__(256) k_rb_spatial(const __grid_constant__ Params p) { RB_XY; spatialPixel<MODE>(p, x, y); }
__global__ void __launch_bounds__(256) k_rb_temporal_accumulation(const __grid_constant__ Params p) { RB_XY; temporalAccumulationPixel(p, x, y); }
__global__ void __launch_bounds__(256) k_rb_history_fix(const __grid_constant__ Params p) { RB_XY; historyFixPixel(p, x, y); }
__global__ void __launch_bounds__(256) k_rb_temporal_stabilization(const __grid_constant__ Params p) { RB_XY; temporalStabilizationPixel(p, x, y); }

} // namespace rb

// 2-D tensor map of a row-major W x H image of `elemBytes`-byte texels with a (24 x boxH) box; false when TMA cannot address the image (pitch or base not 16-byte aligned)
static bool encodeTileMap(CUtensorMap* out, const void* base, uint32_t W, uint32_t H, uint32_t elemBytes, uint32_t boxH)
{
    typedef CUresult (*Encode)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static Encode encode = [] { void* f = nullptr; cudaDriverEntryPointQueryResult q; return (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) ? (Encode)f : (Encode) nullptr; }();
    if (!encode || (size_t(W) * elemBytes) % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15u) != 0) return false;
    const cuuint64_t dims[2] = { W, H }, strides[1] = { cuuint64_t(W) * elemBytes }; const cuuint32_t box[2] = { rb::kHdRegionW, boxH }, estr[2] = { 1, 1 };
    return encode(out, elemBytes == 8 ? CU_TENSOR_MAP_DATA_TYPE_UINT64 : CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int RADIUS> static void launchHitDistReconstruction(const rb::Params& p, bool tiled, dim3 grid, dim3 block, cudaStream_t s)
{
    if (tiled)
    {
        const uint32_t boxH = rb::HitDistRegion<RADIUS>::H;
        rb::HitDistTileMaps maps; memset(&maps, 0, sizeof(maps));
        maps.useTma = (encodeTileMap(&maps.viewZ, p.viewZ, p.W, p.H, 4, boxH) && encodeTileMap(&maps.normalRoughness, p.normalRoughness, p.W, p.H, 4, boxH) && encodeTileMap(&maps.diff, p.inDiff, p.W, p.H, 8, boxH) &&
                       encodeTileMap(&maps.spec, p.inSpec, p.W, p.H, 8, boxH)) ? 1u : 0u;
        rb::k_rb_hit_dist_reconstruction_tiled<RADIUS><<<grid, block, 0, s>>>(p, maps);
    }
    else rb::k_rb_hit_dist_reconstruction<RADIUS><<<grid, block, 0, s>>>(p);
}

void launchReblurFrame(const rb::Params& p, uint32_t hitDistanceReconstructionMode, bool tiled, cudaStream_t s)
{
    const dim3 grid((p.W + 15) / 16, (p.H + 15) / 16), block(16, 16);
    const rb::FrameRouting r = rb::routeFrame(p, hitDistanceReconstructionMode);
    rb::k_rb_classify_tiles<<<grid, block, 0, s>>>(p);
    static const bool envTiled = [] { const char* e = getenv("RTXPT_REBLUR_TILED"); return !e || atoi(e) != 0; }();      // profiling scripts switch a whole process
    if (r.clearSpecTmp1) cudaMemsetAsync(p.tmp1Spec, 0, size_t(p.W) * p.H * sizeof(uint2), s);
    if (r.reconstructionRadius == 2) launchHitDistReconstruction<2>(r.reconstruction, tiled && envTiled, grid, block, s);
    else if (r.reconstructionRadius == 1) launchHitDistReconstruction<1>(r.reconstruction, tiled && envTiled, grid, block, s);
    if (r.prePass) rb::k_rb_spatial<0><<<grid, block, 0, s>>>(r.pre);
    rb::k_rb_temporal_accumulation<<<grid, block, 0, s>>>(r.temporal);
    rb::k_rb_history_fix<<<grid, block, 0, s>>>(p);
    rb::k_rb_spatial<1><<<grid, block, 0, s>>>(p);
    rb::k_rb_spatial<2><<<grid, block, 0, s>>>(p);
    rb::k_rb_temporal_stabilization<<<grid, block, 0, s>>>(p);
}

} // namespace pt
