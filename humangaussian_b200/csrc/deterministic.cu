// deterministic.cu -- the pre-pass and the reduce of the deterministic backward (DESIGN.md section 5, "Deterministic
// backward").  The default B1 adds each (tile, patch) partial into its Gaussian's ScreenGrad record with float REDs, in an
// order that depends on CTA scheduling.  In deterministic mode B1 stores every partial into its own slot instead, and
// det_reduce_kernel adds a Gaussian's partials in a fixed order: its instances in EMISSION order (the tiles of its rect,
// row-major, as emit_tiles_kernel lays them out), within an instance its patches ascending, with sequential fp32 adds.
//   pre-pass: det_start_kernel  start[vp] = offsets_sorted[k] - tiles_touched[vp], vp = order[k]   (one scatter)
//             det_plan_kernel   per (view, tile): the patches' wmax from n_contrib; per sorted instance j of the tile:
//                               pm[j] (bit p = B1 flushes a partial for (j, p), the rule of blend_bwd_kernel) and
//                               jpos[start[vp] + (ty - y0) * w + (tx - x0)] = j
//             lookback_scan     base = inclusive scan of popc(pm), exact 64-bit total H (radix.cuh, via binning.cu)
//   reduce:   det_reduce_kernel one thread per (view, Gaussian): walks its emission range, writes the whole ScreenGrad
//                               record (padding zero), so the default path's scratch memset is not needed
#include "common.cuh"
#include "kernels.h"

DetLayout::DetLayout(int64_t D, int64_t partial_capacity, int64_t n_vp)
{
    const size_t d = (size_t)(D > 0 ? D : 1), cap = (size_t)(partial_capacity > 0 ? partial_capacity : 1),
                 nvp = (size_t)(n_vp > 0 ? n_vp : 1);
    size_t o = 0;
    pm = o; o += gs_align(d);
    base = o; o += gs_align(d * 4);
    jpos = o; o += gs_align(d * 4);
    start = o; o += gs_align(nvp * 4);
    scan_temp = o; o += popc_scan_temp_bytes((int64_t)d);
    total_slot = o; o += 256;
    partials = o; o += gs_align(cap * DET_PARTIAL_FLOATS * sizeof(float));
    total = o;
}

__global__ void __launch_bounds__(256) det_start_kernel(const uint32_t *__restrict__ order, const uint32_t *__restrict__ offsets,
                                                         const uint32_t *__restrict__ tiles_touched, int64_t n_vp,
                                                         uint32_t *__restrict__ start)
{
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_vp) return;
    const uint32_t vp = order[k];
    start[vp] = offsets[k] - tiles_touched[vp];
}

// One 256-thread CTA per (view, tile), thread t <-> pixel t of the tile for the wmax pass, then striding over the tile's list.
__global__ void __launch_bounds__(256) det_plan_kernel(const DetPlanArgs a)
{
    __shared__ int s_wmax[8];
    const int ntiles = a.grid_x * a.grid_y;
    const uint32_t vt = a.tile_order[blockIdx.x];
    const uint2 range = a.ranges[vt];
    if (range.y <= range.x) return; // whole CTA, before any barrier
    const int v = (int)(vt / (uint32_t)ntiles), tile = (int)(vt % (uint32_t)ntiles);
    const int tx = tile % a.grid_x, ty = tile / a.grid_x;
    const int t = threadIdx.x;
    if (t < 8) s_wmax[t] = 0;
    __syncthreads();
    {   // wmax of each 8x4 patch: the largest n_contrib over its in-image pixels, exactly the max B1 forms
        const int lx = t & 15, ly = t >> 4, px = tx * GS_TILE + lx, py = ty * GS_TILE + ly;
        if (px < a.W && py < a.H) {
            const int nc = (int)a.n_contrib[((size_t)v * a.H + py) * a.W + px];
            if (nc > 0) atomicMax(&s_wmax[(ly >> 2) * 2 + (lx >> 3)], nc);
        }
    }
    __syncthreads();
    int lim[8]; // last chunk B1 reads in patch p (-1: none): the chunks c <= (wmax - 1) >> 5 of a patch with wmax > 0
#pragma unroll
    for (int p = 0; p < 8; p++) {
        const int w = s_wmax[p];
        lim[p] = w > 0 ? (w - 1) >> 5 : -1;
    }
    const uint32_t *const cmask = a.cmask + ((size_t)(range.x >> 5) + vt) * 8; // chunk c, patch p: cmask[8c + p]
    for (uint32_t j = range.x + t; j < range.y; j += 256) {
        const uint32_t pos = j - range.x, bit = pos & 31u;
        const int c = (int)(pos >> 5);
        uint32_t m = 0;
#pragma unroll
        for (int p = 0; p < 8; p++)
            if (c <= lim[p]) m |= ((__ldg(cmask + 8 * (size_t)c + p) >> bit) & 1u) << p;
        a.pm[j] = (uint8_t)m;
        const uint32_t vp = a.point_list[j];
        const uint2 r = a.rects[vp];
        const uint32_t x0 = r.x & 0xffff, y0 = r.x >> 16, w = (r.y & 0xffff) - x0;
        const uint32_t e = a.start[vp] + ((uint32_t)ty - y0) * w + ((uint32_t)tx - x0);
        if ((int64_t)e < a.D) a.jpos[e] = j;
    }
}

// One thread per (view, Gaussian), taken in depth order k: vp = order[k] owns the emission indices
// [offsets[k] - tiles_touched[vp], offsets[k]).
__global__ void __launch_bounds__(256) det_reduce_kernel(const DetPlanArgs a, int64_t n_vp, const float *__restrict__ partials,
                                                          float *__restrict__ sgrad)
{
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_vp) return;
    const uint32_t vp = a.order[k];
    const uint32_t n = a.tiles_touched[vp], e0 = a.offsets[k] - n;
    float s[DET_PARTIAL_FLOATS];
#pragma unroll
    for (int i = 0; i < DET_PARTIAL_FLOATS; i++) s[i] = 0.0f;
    for (uint32_t e = e0; e != e0 + n; e++) {
        const uint32_t j = __ldg(a.jpos + e);
        const uint32_t np = (uint32_t)__popc((uint32_t)__ldg(a.pm + j));
        const uint32_t end = __ldg(a.base + j); // partials [end - np, end), patches ascending
        for (uint32_t q = end - np; q != end; q++) {
            const float2 *r = reinterpret_cast<const float2 *>(partials + (size_t)q * DET_PARTIAL_FLOATS);
#pragma unroll
            for (int i = 0; i < DET_PARTIAL_FLOATS / 2; i++) {
                const float2 x = __ldg(r + i);
                s[2 * i] = fadd(s[2 * i], x.x);
                s[2 * i + 1] = fadd(s[2 * i + 1], x.y);
            }
        }
    }
    float4 *dst = reinterpret_cast<float4 *>(sgrad + (size_t)vp * (sizeof(ScreenGrad) / sizeof(float)));
    dst[0] = make_float4(s[0], s[1], s[2], s[3]);
    dst[1] = make_float4(s[4], s[5], s[6], s[7]);
    dst[2] = make_float4(s[8], s[9], 0.0f, 0.0f);
}

int launch_det_plan(const DetPlanArgs &a, int64_t n_vp, int n_tiles_all, const DetLayout &L, char *det_base, cudaStream_t st,
                    int *n_launches)
{
    det_start_kernel<<<(unsigned)((n_vp + 255) / 256), 256, 0, st>>>(a.order, a.offsets, a.tiles_touched, n_vp, a.start);
    det_plan_kernel<<<(unsigned)n_tiles_all, 256, 0, st>>>(a);
    *n_launches += 3;
    return launch_popc_scan(a.pm, a.base, a.D, det_base + L.scan_temp, (uint64_t *)(det_base + L.total_slot), st);
}

void launch_det_reduce(const DetPlanArgs &a, int64_t n_vp, const float *partials, void *sgrad, cudaStream_t st)
{
    det_reduce_kernel<<<(unsigned)((n_vp + 255) / 256), 256, 0, st>>>(a, n_vp, partials, (float *)sgrad);
}
