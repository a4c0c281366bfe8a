// radix.cuh -- hand-written stable LSD radix sort of (key, u32 value) pairs and a decoupled-look-back scan,
// the two primitives of the binning stage (SURVEY.md Appendix A.3).  sm_90a, 256-thread CTAs.
//
// One pass = count (per-CTA digit histogram) -> scan over CTAs -> ranked scatter: every CTA ranks its tile of
// 256*IPT items by digit with warp match.any + per-warp shared counters (stable: items keep their input order
// inside a digit), reorders the tile through shared memory so that the final global stores are contiguous runs
// per digit, and scatters to destinations taken from the scanned counts.  Digit width is a template parameter
// (6..9 bits): the tile-key sort of a 64-view batch (18 bits) takes 2 passes of 9 bits where an 8-bit library
// sort takes 3.  The scan over tiles_touched uses a decoupled look-back (one word per CTA, short walks).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsradix {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

template <typename KeyT>
__device__ __forceinline__ uint32_t digit_of(KeyT k, int shift, int bits)
{
    return (uint32_t)(k >> shift) & ((1u << bits) - 1u);
}

// ---- pass = three kernels: per-CTA digit counts -> scan over CTAs -> ranked scatter -------------------------------
// (A single-kernel "onesweep" with decoupled look-back was tried first: with 512 digits every CTA needs 512
//  independent look-back walks, and with ~740 CTAs in flight the walks are hundreds of dependent L2 round trips
//  deep -- it ran at 1.2 TB/s.  Counting first costs one extra read of the keys and removes every spin.)

// counts[d][cta] = number of items of CTA `cta` whose digit is d          (digit-major: the scan is contiguous)
template <typename KeyT, int RADIX_BITS, int IPT>
__global__ void __launch_bounds__(THREADS) count_kernel(const KeyT *__restrict__ keys, int64_t n, const uint64_t *__restrict__ n_dev, int shift, int bits,
                                                         uint32_t *__restrict__ counts, uint32_t nblocks)
{
    // n_dev (optional): the item count lives on the device (the host sized the grid for the capacity `n` without waiting for
    // it); CTAs past the real count write zero counts and do nothing else
    if (n_dev) n = min(n, (int64_t)*n_dev);
    constexpr int BINS = 1 << RADIX_BITS;
    constexpr int TILE = THREADS * IPT;
    __shared__ uint32_t sh[BINS];
    for (int i = threadIdx.x; i < BINS; i += THREADS) sh[i] = 0;
    __syncthreads();
    const int64_t tile_start = (int64_t)blockIdx.x * TILE;
    const int n_tile = (int)min((int64_t)TILE, n - tile_start);
    KeyT key[IPT];
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        const int idx = i * THREADS + threadIdx.x;
        key[i] = (idx < n_tile) ? keys[tile_start + idx] : (KeyT)0;
    }
#pragma unroll
    for (int i = 0; i < IPT; i++)
        if (i * THREADS + (int)threadIdx.x < n_tile) atomicAdd(&sh[digit_of(key[i], shift, bits)], 1u);
    __syncthreads();
    for (int i = threadIdx.x; i < BINS; i += THREADS) counts[(size_t)i * nblocks + blockIdx.x] = sh[i];
}

// one CTA per digit: exclusive scan of its row of per-CTA counts in place; totals[d] = row sum.
// The row is walked in slabs of 4 * THREADS consecutive counts (four per thread: neighbouring lanes touch neighbouring
// 16-byte groups) with one block scan per slab and a running carry.  (Round 1 gave every thread one contiguous chunk of the
// row: lane-to-lane stride of `nblocks / 256` words, 47 us per launch on the 64-view step, six launches per step.)
__global__ void __launch_bounds__(THREADS) scan_counts_kernel(uint32_t *__restrict__ counts, uint32_t nblocks, uint32_t *__restrict__ totals)
{
    __shared__ uint32_t s_wsum[2][WARPS];
    uint32_t *row = counts + (size_t)blockIdx.x * nblocks;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint32_t carry = 0;
    int buf = 0;
    for (uint32_t base = 0; base < nblocks; base += 4 * THREADS, buf ^= 1) {
        const uint32_t i0 = base + 4 * (uint32_t)tid;
        uint32_t c[4];
#pragma unroll
        for (int j = 0; j < 4; j++) c[j] = (i0 + j < nblocks) ? row[i0 + j] : 0u;
        const uint32_t tsum = c[0] + c[1] + c[2] + c[3];
        uint32_t incl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_wsum[buf][warp] = incl;
        __syncthreads(); // one barrier per slab: the warp sums are double buffered
        uint32_t wbase = 0, total = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) {
            const uint32_t x = s_wsum[buf][w];
            if (w < warp) wbase += x;
            total += x;
        }
        uint32_t run = carry + wbase + incl - tsum;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (i0 + j < nblocks) row[i0 + j] = run;
            run += c[j];
        }
        carry += total;
    }
    if (tid == 0) totals[blockIdx.x] = carry;
}

// ranked scatter of one CTA tile: stable inside the tile, destinations from the scanned counts
template <typename KeyT, int RADIX_BITS, int IPT>
__global__ void __launch_bounds__(THREADS) scatter_kernel(const KeyT *__restrict__ keys_in, KeyT *__restrict__ keys_out,
                                                           const uint32_t *__restrict__ vals_in, uint32_t *__restrict__ vals_out,
                                                           int64_t n, const uint64_t *__restrict__ n_dev, int shift, int bits,
                                                           const uint32_t *__restrict__ counts /* scanned */, uint32_t nblocks,
                                                           const uint32_t *__restrict__ totals)
{
    if (n_dev) n = min(n, (int64_t)*n_dev);
    if ((int64_t)blockIdx.x * (THREADS * IPT) >= n) return; // a CTA past the device-side count (whole CTA: no barrier is skipped)
    constexpr int BINS = 1 << RADIX_BITS;
    constexpr int TILE = THREADS * IPT;
    constexpr int DPT = (BINS + THREADS - 1) / THREADS; // digits per thread in the per-digit phases
    __shared__ uint32_t s_cnt[WARPS][BINS]; // per-warp digit counters -> exclusive warp prefixes
    __shared__ uint32_t s_loc[BINS];        // exclusive scan of the CTA's digit counts (local sorted offsets)
    __shared__ uint32_t s_glob[BINS];       // global destination of the CTA's first item of each digit
    __shared__ KeyT s_keys[TILE];
    __shared__ uint32_t s_vals[TILE];
    __shared__ uint32_t s_wsum[WARPS];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t bid = blockIdx.x;
    for (int i = tid; i < WARPS * BINS; i += THREADS) (&s_cnt[0][0])[i] = 0;
    const int64_t tile_start = (int64_t)bid * TILE;
    const int n_tile = (int)min((int64_t)TILE, n - tile_start);

    // ---- load (warp-striped: coalesced); all loads are issued before the first use
    KeyT key[IPT];
    uint32_t val[IPT], rnk[IPT];
    const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        const int idx = warp * (IPT * 32) + i * 32 + lane;
        key[i] = (idx < n_tile) ? keys_in[tile_start + idx] : (KeyT)0;
    }
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        const int idx = warp * (IPT * 32) + i * 32 + lane;
        val[i] = (idx < n_tile) ? vals_in[tile_start + idx] : 0u;
    }
    // digit totals -> (later) global digit bases
    uint32_t tot[DPT], cnt_glob[DPT];
#pragma unroll
    for (int q = 0; q < DPT; q++) {
        const int d = tid + q * THREADS;
        tot[q] = (d < BINS) ? totals[d] : 0u;
        cnt_glob[q] = (d < BINS) ? counts[(size_t)d * nblocks + bid] : 0u;
    }
    __syncthreads();
    // ---- rank: stable position of every item among the items of its digit inside this warp
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        const int idx = warp * (IPT * 32) + i * 32 + lane;
        const bool valid = idx < n_tile;
        const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
        rnk[i] = 0xffffffffu;
        if (valid) {
            const uint32_t d = digit_of(key[i], shift, bits);
            const uint32_t peers = __match_any_sync(vmask, d);
            const uint32_t before = s_cnt[warp][d];
            __syncwarp(vmask);
            if ((peers & lt) == 0) s_cnt[warp][d] = before + __popc(peers);
            __syncwarp(vmask);
            rnk[i] = before + __popc(peers & lt);
        }
    }
    __syncthreads();
    // ---- per digit: exclusive prefix over warps, CTA count
    uint32_t cta_count[DPT];
#pragma unroll
    for (int q = 0; q < DPT; q++) {
        const int d = tid + q * THREADS;
        cta_count[q] = 0;
        if (d < BINS) {
            uint32_t run = 0;
#pragma unroll
            for (int w = 0; w < WARPS; w++) {
                const uint32_t c = s_cnt[w][d];
                s_cnt[w][d] = run;
                run += c;
            }
            cta_count[q] = run;
        }
    }
    // ---- two exclusive scans over digits (digits are spread tid + q*THREADS): local offsets and global bases
    {
        uint32_t slab_base_l = 0, slab_base_g = 0;
#pragma unroll
        for (int q = 0; q < DPT; q++) {
            uint32_t il = cta_count[q], ig = tot[q];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t yl = __shfl_up_sync(0xffffffffu, il, o), yg = __shfl_up_sync(0xffffffffu, ig, o);
                if (lane >= o) { il += yl; ig += yg; }
            }
            __syncthreads();
            if (lane == 31) s_wsum[warp] = il;
            __syncthreads();
            uint32_t wl = 0, tl = 0;
            for (int w = 0; w < WARPS; w++) { if (w < warp) wl += s_wsum[w]; tl += s_wsum[w]; }
            __syncthreads();
            if (lane == 31) s_wsum[warp] = ig;
            __syncthreads();
            uint32_t wg = 0, tg = 0;
            for (int w = 0; w < WARPS; w++) { if (w < warp) wg += s_wsum[w]; tg += s_wsum[w]; }
            const int d = tid + q * THREADS;
            if (d < BINS) {
                s_loc[d] = slab_base_l + wl + il - cta_count[q];
                s_glob[d] = slab_base_g + wg + ig - tot[q] + cnt_glob[q];
            }
            slab_base_l += tl;
            slab_base_g += tg;
        }
    }
    __syncthreads();

    // ---- reorder through shared memory (local stable sort by digit), then scatter contiguous runs
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        if (rnk[i] != 0xffffffffu) {
            const uint32_t d = digit_of(key[i], shift, bits);
            const uint32_t lpos = s_loc[d] + s_cnt[warp][d] + rnk[i];
            s_keys[lpos] = key[i];
            s_vals[lpos] = val[i];
        }
    }
    __syncthreads();
    for (int k = tid; k < n_tile; k += THREADS) {
        const KeyT kk = s_keys[k];
        const uint32_t d = digit_of(kk, shift, bits);
        const int64_t dst = (int64_t)s_glob[d] + (k - s_loc[d]);
        keys_out[dst] = kk;
        vals_out[dst] = s_vals[k];
    }
}

// ---- inclusive scan of x[k] = load(k) with decoupled look-back (single pass over the data) ------------
// Loads: the binning stage scans tiles_touched in depth order (GatherLoad); the deterministic backward scans the partial
// counts popc(pm[j]) of the sorted instances (PopcLoad, deterministic.cu).
constexpr int SCAN_IPT = 8;
struct GatherLoad { // x[k] = tiles[order[k]]
    const uint32_t *order, *tiles;
    __device__ __forceinline__ uint32_t operator()(int64_t k) const { return __ldg(tiles + __ldg(order + k)); }
};
template <typename Load>
__global__ void __launch_bounds__(THREADS) lookback_scan_kernel(const Load load, uint32_t *__restrict__ out, int64_t n,
                                                                 volatile uint64_t *status /* [nblocks], zeroed */,
                                                                 uint32_t *ticket /* zeroed */, uint64_t *total_out /* exact 64-bit sum */)
{
    // status: bit 63 = prefix ready, bit 62 = aggregate ready, low 56 bits = value (the exact running sum: fewer than 2^32
    // entries of at most 2^24 each cannot reach 2^56).  out[] keeps the low 32 bits; the callers check the exact total before
    // anything relies on the 32-bit values (api.cu).
    constexpr int TILE = THREADS * SCAN_IPT;
    __shared__ uint32_t s_bid, s_wsum[WARPS];
    __shared__ uint64_t s_excl;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) s_bid = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t bid = s_bid;
    const int64_t base = (int64_t)bid * TILE + (int64_t)tid * SCAN_IPT;
    uint32_t x[SCAN_IPT];
    uint32_t tsum = 0;
#pragma unroll
    for (int i = 0; i < SCAN_IPT; i++) {
        x[i] = (base + i < n) ? load(base + i) : 0u;
        tsum += x[i];
    }
    uint32_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0, total = 0;
    for (int w = 0; w < WARPS; w++) {
        if (w < warp) wbase += s_wsum[w];
        total += s_wsum[w];
    }
    if (tid == 0) {
        const uint64_t AGG = 1ull << 62, PRE = 1ull << 63, VM = (1ull << 56) - 1;
        status[bid] = (bid == 0 ? PRE : AGG) | (uint64_t)total;
        __threadfence();
        uint64_t excl = 0;
        if (bid > 0) {
            int64_t p = (int64_t)bid - 1;
            while (true) {
                uint64_t s;
                do { s = status[p]; } while ((s >> 62) == 0);
                excl += s & VM;
                if (s & PRE) break;
                p--;
            }
            status[bid] = PRE | (excl + total);
        }
        if ((int64_t)(bid + 1) * TILE >= n) *total_out = excl + total; // the block holding the last element
        s_excl = excl;
    }
    __syncthreads();
    uint32_t run = (uint32_t)s_excl + wbase + incl - tsum;
#pragma unroll
    for (int i = 0; i < SCAN_IPT; i++) {
        run += x[i];
        if (base + i < n) out[base + i] = run;
    }
}

} // namespace gsradix
