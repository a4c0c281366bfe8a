// binning.cu -- F2..F5 (SURVEY.md Appendix A.3) re-designed around a DEPTH PRE-SORT, all kernels hand-written.
//
// Upstream sorts D = sum(tiles_touched) 64-bit (tile|depth) keys: ~7 radix passes over every (Gaussian, tile)
// instance.  The order it defines -- inside each tile ascending depth, ties by ascending Gaussian index -- is
// reproduced here with far less traffic:
//   1. sort the V*P Gaussians once by depth bits (all views mixed: step 4's key carries the view)
//                                                          [stable LSD radix, 4 passes of 8-bit digits on 4-byte keys; V*P is 4-5x smaller than D]
//   2. inclusive scan of tiles_touched IN THAT ORDER        [single-pass decoupled look-back] -> D and emission offsets
//   3. emit instances in depth order: key = view*tiles + tile (32 bit), value = record index
//   4. STABLE sort by the tile key only                     [9-bit digits: 2 passes for 12..18 bits, 8-byte pairs]
//   5. tile ranges from the sorted tile keys
// Stability of step 4 keeps step 1's (depth, index) order inside every tile, so point_list and ranges are
// bit-identical to the reference's single 64-bit sort (tests compare them, and the reconstructed 64-bit keys,
// against the oracle).  The sort (count / scan / ranked-scatter passes) and the look-back scan are in radix.cuh.
#include "common.cuh"
#include "kernels.h"
#include "radix.cuh"

using namespace gsradix;

static int bits_for(uint64_t n)
{
    int b = 0;
    while (((uint64_t)1 << b) < n) b++;
    return b;
}

// sort configuration
constexpr int D_BITS = 8, D_IPT = 12, D_TILE = THREADS * D_IPT;   // depth sort: u32 keys (the depth bits)
constexpr int T_BITS = 9, T_IPT = 12, T_TILE = THREADS * T_IPT;   // tile sort: u32 keys
constexpr int MAXP = 5;
constexpr int SCAN_TILE = THREADS * SCAN_IPT;
// The depth order is read from order_in after the pre-sort by the deterministic backward's plan (api.cu, backward_impl)
// and by b200gs_describe_state: right only when the ping-pong passes end in the buffer they started from.
static_assert(((32 + D_BITS - 1) / D_BITS) % 2 == 0,
              "odd depth pre-sort pass count: the depth order ends in BinLayout::order, so backward_impl's pa.order and "
              "b200gs_describe_state's depth_order (api.cu) must read it there instead of order_in");

// scratch of one radix sort: digit totals + the [digit][CTA] count matrix (re-used by every pass)
static size_t sort_scratch_bytes(int64_t n, int tile, int bins)
{
    const size_t nblocks = (size_t)((n + tile - 1) / tile) + 1;
    return gs_align((size_t)bins * 4) + gs_align(nblocks * bins * 4);
}

BinLayout binning_layout(int64_t capacity, int ntiles_total, int64_t n_vp)
{
    BinLayout L;
    const size_t cap = (size_t)(capacity > 0 ? capacity : 1), nvp = (size_t)(n_vp > 0 ? n_vp : 1);
    size_t o = 0;
    L.keys_in = o; o += gs_align(cap * 4);
    L.keys_out = o; o += gs_align(cap * 4);
    L.vals_in = o; o += gs_align(cap * 4);
    L.vals_out = o; o += gs_align(cap * 4);
    L.ranges = o; o += gs_align((size_t)ntiles_total * 8);
    L.dkeys_in = o; o += gs_align(nvp * 4);
    L.dkeys_out = o; o += gs_align(nvp * 4);
    L.order_in = o; o += gs_align(nvp * 4);
    L.order = o; o += gs_align(nvp * 4);
    L.tile_order = o; o += gs_align((size_t)ntiles_total * 4);
    L.tile_order_cnt = o; o += gs_align(64 * 4);
    L.total_slot = o; o += 256; // the scan's exact 64-bit instance count: read by the later kernels, so NOT inside the re-used temp area
    L.cmask = o; o += gs_align(((cap >> 5) + (size_t)ntiles_total + 1) * 8 * 4);
    const size_t s_depth = sort_scratch_bytes((int64_t)nvp, D_TILE, 1 << D_BITS);
    const size_t s_tile = sort_scratch_bytes((int64_t)cap, T_TILE, 1 << T_BITS);
    const size_t s_scan = gs_align(((nvp + SCAN_TILE - 1) / SCAN_TILE + 1) * 8) + 256;
    size_t t = s_depth > s_tile ? s_depth : s_tile;
    t = t > s_scan ? t : s_scan;
    L.temp_bytes = t;
    L.temp = o; o += L.temp_bytes;
    L.total = o;
    return L;
}

// Generic driver: stable LSD radix sort of n pairs over key bits [0, nbits).  Buffers a/b ping-pong; on return
// *keys_sorted / *vals_sorted point at whichever buffer holds the result.  scratch must be sort_scratch_bytes().
template <typename KeyT, int RBITS, int IPT>
static int radix_sort_pairs(KeyT *ka, KeyT *kb, uint32_t *va, uint32_t *vb, int64_t n, const uint64_t *n_dev, int nbits, char *scratch,
                            size_t scratch_bytes, KeyT **keys_sorted, uint32_t **vals_sorted, cudaStream_t st, int *n_launches)
{
    constexpr int BINS = 1 << RBITS, TILE = THREADS * IPT;
    if (nbits < 1) nbits = 1;
    const int npass = (nbits + RBITS - 1) / RBITS;
    if (npass > MAXP) return -1;
    const int last_bits = nbits - (npass - 1) * RBITS;
    const uint32_t nblocks = (uint32_t)((n + TILE - 1) / TILE);
    uint32_t *totals = (uint32_t *)scratch;
    uint32_t *counts = (uint32_t *)(scratch + gs_align((size_t)BINS * 4));
    if (gs_align((size_t)BINS * 4) + (size_t)nblocks * BINS * 4 > scratch_bytes) return -2;
    KeyT *kin = ka, *kout = kb;
    uint32_t *vin = va, *vout = vb;
    for (int p = 0; p < npass; p++) {
        const int bits = (p == npass - 1) ? last_bits : RBITS;
        count_kernel<KeyT, RBITS, IPT><<<nblocks, THREADS, 0, st>>>(kin, n, n_dev, p * RBITS, bits, counts, nblocks);
        scan_counts_kernel<<<BINS, THREADS, 0, st>>>(counts, nblocks, totals);
        scatter_kernel<KeyT, RBITS, IPT><<<nblocks, THREADS, 0, st>>>(kin, kout, vin, vout, n, n_dev, p * RBITS, bits, counts, nblocks, totals);
        KeyT *tk = kin; kin = kout; kout = tk;
        uint32_t *tv = vin; vin = vout; vout = tv;
    }
    *keys_sorted = kin;
    *vals_sorted = vin;
    *n_launches += 3 * npass;
    return 0;
}

// depth pre-sort + scan in depth order.  dkeys_in / order_in were written by the preprocess kernel.
// On return *order_sorted points at the sorted record indices (inside bin_base) and *total_dev at the exact 64-bit
// instance count of the batch (device word, valid once the stream reaches this point).
int launch_depth_order(const uint32_t *tiles_touched, uint32_t *offsets_sorted, int64_t n_vp, int V, char *bin_base,
                       const BinLayout &L, const uint32_t **order_sorted, const uint64_t **total_dev, cudaStream_t st, int *n_launches)
{
    uint32_t *ks = nullptr, *vs = nullptr;
    if (radix_sort_pairs<uint32_t, D_BITS, D_IPT>((uint32_t *)(bin_base + L.dkeys_in), (uint32_t *)(bin_base + L.dkeys_out),
                                                  (uint32_t *)(bin_base + L.order_in), (uint32_t *)(bin_base + L.order), n_vp,
                                                  nullptr, 32, bin_base + L.temp, L.temp_bytes, &ks, &vs, st, n_launches))
        return -1;
    *order_sorted = vs;
    const size_t nblocks = (size_t)((n_vp + SCAN_TILE - 1) / SCAN_TILE);
    char *scr = bin_base + L.temp;
    cudaMemsetAsync(scr, 0, gs_align((nblocks + 1) * 8) + 256, st);
    lookback_scan_kernel<<<(unsigned)nblocks, THREADS, 0, st>>>(GatherLoad{vs, tiles_touched}, offsets_sorted, n_vp,
                                                               (volatile uint64_t *)(scr + 256), (uint32_t *)scr,
                                                               (uint64_t *)(bin_base + L.total_slot));
    *total_dev = (const uint64_t *)(bin_base + L.total_slot);
    *n_launches += 1;
    return cudaPeekAtLastError() == cudaSuccess ? 0 : -2;
}

// The deterministic backward's partial counts: x[j] = popc(pm[j]), scanned with the same look-back kernel
struct PopcLoad {
    const uint8_t *pm;
    __device__ __forceinline__ uint32_t operator()(int64_t j) const { return (uint32_t)__popc((uint32_t)__ldg(pm + j)); }
};
size_t popc_scan_temp_bytes(int64_t n) { return 256 + gs_align((size_t)((n + SCAN_TILE - 1) / SCAN_TILE + 1) * 8); }
int launch_popc_scan(const uint8_t *pm, uint32_t *incl, int64_t n, char *temp, uint64_t *total, cudaStream_t st)
{
    if (n < 1) return -1;
    if (cudaMemsetAsync(temp, 0, popc_scan_temp_bytes(n), st) != cudaSuccess) return -1;
    lookback_scan_kernel<<<(unsigned)((n + SCAN_TILE - 1) / SCAN_TILE), THREADS, 0, st>>>(PopcLoad{pm}, incl, n,
                                                                                        (volatile uint64_t *)(temp + 256),
                                                                                        (uint32_t *)temp, total);
    return cudaPeekAtLastError() == cudaSuccess ? 0 : -1;
}

// Instance emission, warp-cooperative.  A warp owns 32 consecutive Gaussians IN DEPTH ORDER; their instances form one
// contiguous run [start of lane 0, end of lane 31) of the output, so lane j writes output element base+j (fully coalesced
// 128-byte stores) after finding its owner Gaussian with a 5-step shuffle binary search over the 32 run starts.
// (A thread-per-Gaussian loop writes 4-byte words 18 bytes apart on average: uncoalesced.)
__global__ void __launch_bounds__(256) emit_tiles_kernel(const uint32_t *__restrict__ order, const uint2 *__restrict__ rects,
                                                          const uint32_t *__restrict__ offsets_sorted, int P, int64_t n_vp,
                                                          int grid_x, int ntiles, uint32_t cap, uint32_t *__restrict__ keys,
                                                          uint32_t *__restrict__ vals)
{   // cap: capacity of keys/vals.  The host launches this before it knows the instance count; if the batch turns out larger
    // than the capacity the writes stop at cap (the call then reports B200GS_E_BIN_TOO_SMALL and is repeated with more room)
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t vp = 0, x0 = 0, y0 = 0, w = 1, cnt = 0, end = 0;
    if (k < n_vp) {
        vp = order[k];
        const uint2 r = rects[vp];
        const uint32_t rx0 = r.x & 0xffff, ry0 = r.x >> 16, rx1 = r.y & 0xffff, ry1 = r.y >> 16;
        end = offsets_sorted[k];
        if (rx1 > rx0 && ry1 > ry0) { x0 = rx0; y0 = ry0; w = rx1 - rx0; cnt = w * (ry1 - ry0); }
    }
    // lanes past n_vp: empty runs starting where the last valid lane ends
    const int64_t k_last = n_vp - 1;
    const int last_valid = (int)min((int64_t)31, k_last - (k - lane));
    end = __shfl_sync(0xffffffffu, end, min(lane, last_valid));
    if (k >= n_vp) cnt = 0;
    const uint32_t start = end - cnt;
    const uint32_t tile_base = (vp / (uint32_t)P) * (uint32_t)ntiles + y0 * (uint32_t)grid_x + x0;
    const uint32_t warp_start = __shfl_sync(0xffffffffu, start, 0), warp_end = __shfl_sync(0xffffffffu, end, 31);
    for (uint32_t base = warp_start; base < warp_end; base += 32) {
        const uint32_t j = base + lane;
        int lo = 0; // largest lane whose run starts at or before j (empty runs share their successor's start, so the
                    // last lane with that start is the one that owns j)
#pragma unroll
        for (int step = 16; step >= 1; step >>= 1) {
            const uint32_t s = __shfl_sync(0xffffffffu, start, (lo + step) & 31);
            if (lo + step < 32 && s <= j) lo += step;
        }
        const uint32_t o_start = __shfl_sync(0xffffffffu, start, lo);
        const uint32_t o_w = __shfl_sync(0xffffffffu, w, lo);
        const uint32_t o_base = __shfl_sync(0xffffffffu, tile_base, lo);
        const uint32_t o_vp = __shfl_sync(0xffffffffu, vp, lo);
        if (j < warp_end && j < cap) {
            const uint32_t local = j - o_start;
            const uint32_t dy = local / o_w, dx = local - dy * o_w;
            keys[j] = o_base + dy * (uint32_t)grid_x + dx;
            vals[j] = o_vp;
        }
    }
}

// tile boundaries of the sorted keys: four keys per thread (one 128-bit load + the neighbour before)
__global__ void __launch_bounds__(256) tile_ranges_kernel(const uint32_t *__restrict__ keys, int64_t D, const uint64_t *__restrict__ D_dev,
                                                           uint2 *__restrict__ ranges)
{
    if (D_dev) D = min(D, (int64_t)*D_dev);
    const int64_t j0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (j0 >= D) return;
    uint32_t t[4];
    if (j0 + 3 < D) {
        const uint4 q = *reinterpret_cast<const uint4 *>(keys + j0);
        t[0] = q.x; t[1] = q.y; t[2] = q.z; t[3] = q.w;
    } else {
        for (int i = 0; i < 4; i++) t[i] = (j0 + i < D) ? keys[j0 + i] : 0u;
    }
    uint32_t prev = (j0 == 0) ? 0u : keys[j0 - 1];
    if (j0 == 0) ranges[t[0]].x = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int64_t j = j0 + i;
        if (j < D) {
            if (j > 0 && prev != t[i]) {
                ranges[prev].y = (uint32_t)j;
                ranges[t[i]].x = (uint32_t)j;
            }
            if (j == D - 1) ranges[t[i]].y = (uint32_t)D;
            prev = t[i];
        }
    }
}

// ---- launch order of the tiles: longest list first (LPT).  One view is otherwise bounded by its heaviest tiles being
// dispatched in the middle of the grid; results do not depend on this order.  Buckets = floor(log2(length)) + 1.
__global__ void __launch_bounds__(256) tile_bucket_count_kernel(const uint2 *__restrict__ ranges, int n, uint32_t *__restrict__ cnt)
{
    __shared__ uint32_t sh[32];
    if (threadIdx.x < 32) sh[threadIdx.x] = 0;
    __syncthreads();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) {
        const uint2 r = ranges[t];
        atomicAdd(&sh[32 - __clz(r.y - r.x)], 1u); // length 0 -> bucket 0, 1 -> 1, 2..3 -> 2, ...
    }
    __syncthreads();
    if (threadIdx.x < 32 && sh[threadIdx.x]) atomicAdd(&cnt[threadIdx.x], sh[threadIdx.x]);
}
__global__ void __launch_bounds__(256) tile_bucket_scatter_kernel(const uint2 *__restrict__ ranges, int n, uint32_t *__restrict__ cnt /* [0,32): counts, [32,64): cursors */,
                                                                   uint32_t *__restrict__ order)
{
    __shared__ uint32_t s_base[32], s_local[32];
    if (threadIdx.x < 32) s_local[threadIdx.x] = 0;
    __syncthreads();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int b = 0;
    uint32_t my = 0;
    if (t < n) {
        const uint2 r = ranges[t];
        b = 32 - __clz(r.y - r.x);
        my = atomicAdd(&s_local[b], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        // descending buckets: start of bucket k = sum of counts of buckets > k ; claim this CTA's slice with one atomic
        uint32_t start = 0;
        for (int k = 31; k > (int)threadIdx.x; k--) start += cnt[k];
        s_base[threadIdx.x] = s_local[threadIdx.x] ? start + atomicAdd(&cnt[32 + threadIdx.x], s_local[threadIdx.x]) : 0u;
    }
    __syncthreads();
    if (t < n) order[s_base[b] + my] = (uint32_t)t;
}

// After this call the sorted tile keys are at bin_base+L.keys_out and the point list at bin_base+L.vals_out
// (a device-to-device copy fixes the parity when the number of passes is even).
// D: the instance count if the host knows it (D_dev == nullptr), else the CAPACITY the launches are sized for while the real
// count is read by the kernels from *D_dev (no host synchronisation between the scan and the sort).
int launch_binning(const uint32_t *order_sorted, const uint2 *rects, const uint32_t *offsets_sorted, int P, int V, int grid_x, int grid_y,
                   int64_t D, const uint64_t *D_dev, char *bin_base, const BinLayout &L, cudaStream_t st, int *n_launches)
{
    const int ntiles = grid_x * grid_y;
    const int64_t n_vp = (int64_t)P * V;
    uint32_t *keys_in = (uint32_t *)(bin_base + L.keys_in), *keys_out = (uint32_t *)(bin_base + L.keys_out);
    uint32_t *vals_in = (uint32_t *)(bin_base + L.vals_in), *vals_out = (uint32_t *)(bin_base + L.vals_out);
    uint2 *ranges = (uint2 *)(bin_base + L.ranges);
    cudaMemsetAsync(ranges, 0, (size_t)ntiles * V * 8, st);
    uint32_t *tile_order = (uint32_t *)(bin_base + L.tile_order), *tcnt = (uint32_t *)(bin_base + L.tile_order_cnt);
    const int nt_all = ntiles * V;
    if (D == 0 && !D_dev) { // every list is empty (count known on the host): identity order
        cudaMemsetAsync(tcnt, 0, 64 * 4, st);
        tile_bucket_count_kernel<<<(nt_all + 255) / 256, 256, 0, st>>>(ranges, nt_all, tcnt);
        tile_bucket_scatter_kernel<<<(nt_all + 255) / 256, 256, 0, st>>>(ranges, nt_all, tcnt, tile_order);
        *n_launches += 2;
        return 0;
    }
    if (D > B200GS_MAX_INSTANCES_I64) return -3; // api.cu rejects this before calling; 32-bit instance indices end here
    const int nbits = bits_for((uint64_t)ntiles * V) > 0 ? bits_for((uint64_t)ntiles * V) : 1;
    const int npass = (nbits + T_BITS - 1) / T_BITS;
    // emit into the buffer from which `npass` ping-pong passes end in keys_out/vals_out
    uint32_t *k0 = (npass & 1) ? keys_in : keys_out, *k1 = (npass & 1) ? keys_out : keys_in;
    uint32_t *v0 = (npass & 1) ? vals_in : vals_out, *v1 = (npass & 1) ? vals_out : vals_in;
    emit_tiles_kernel<<<(unsigned)((n_vp + 255) / 256), 256, 0, st>>>(order_sorted, rects, offsets_sorted, P, n_vp, grid_x, ntiles, (uint32_t)D, k0, v0);
    uint32_t *ks = nullptr, *vs = nullptr;
    if (radix_sort_pairs<uint32_t, T_BITS, T_IPT>(k0, k1, v0, v1, D, D_dev, nbits, bin_base + L.temp, L.temp_bytes, &ks, &vs, st, n_launches)) return -2;
    if (ks != keys_out || vs != vals_out) return -4;
    tile_ranges_kernel<<<(unsigned)((D + 1023) / 1024), 256, 0, st>>>(keys_out, D, D_dev, ranges);
    cudaMemsetAsync(tcnt, 0, 64 * 4, st);
    tile_bucket_count_kernel<<<(nt_all + 255) / 256, 256, 0, st>>>(ranges, nt_all, tcnt);
    tile_bucket_scatter_kernel<<<(nt_all + 255) / 256, 256, 0, st>>>(ranges, nt_all, tcnt, tile_order);
    *n_launches += 4;
    return 0;
}

// test hook: sort n (u32 key, u32 value) pairs stably over the low nbits of the key with the tile-sort kernels
int launch_test_sort32(uint32_t *ka, uint32_t *kb, uint32_t *va, uint32_t *vb, int64_t n, int nbits, char *scratch, size_t scratch_bytes,
                       int *result_in_b, cudaStream_t st)
{
    uint32_t *ks = nullptr, *vs = nullptr;
    int nl = 0;
    const int rc = radix_sort_pairs<uint32_t, T_BITS, T_IPT>(ka, kb, va, vb, n, nullptr, nbits, scratch, scratch_bytes, &ks, &vs, st, &nl);
    *result_in_b = (ks == kb);
    return rc;
}
size_t test_sort32_scratch_bytes(int64_t n) { return sort_scratch_bytes(n, T_TILE, 1 << T_BITS); }
