// Device primitives shared by the broad phase, the contact graph and the spatial queries: the stable LSD radix-sort pass (8-bit digits, 2048 keys
// per block), the exclusive scan of per-item counts into CSR offsets and the open-addressing u64 hash set.  Everything lives in an anonymous namespace: each translation unit that includes this gets its own copies.
#pragma once
#include <cstdint>

namespace avn {
namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ROUNDS = 8;                       // elements per thread per tile
constexpr int RS_TILE = RS_THREADS * RS_ROUNDS;    // 2048 keys per block

// digit histogram of one tile -> hist[digit * nblocks + block]
template <class K>
__global__ void __launch_bounds__(RS_THREADS) rs_histogram(const K* __restrict__ keys, int n, int shift, uint32_t* __restrict__ hist, int nblocks) {
    __shared__ uint32_t cnt[256];
    cnt[threadIdx.x] = 0;
    __syncthreads();
    const int base = blockIdx.x * RS_TILE;
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        int i = base + r * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&cnt[(keys[i] >> shift) & 0xff], 1u);
    }
    __syncthreads();
    hist[threadIdx.x * nblocks + blockIdx.x] = cnt[threadIdx.x];
}

// exclusive scan of `len` counters by one block (len = 256 * nblocks: 12 544 for 100k keys, 125 184 for 1M).  Each thread owns
// RS_SCAN_ITEMS consecutive counters per iteration (serial sum, block scan of the sums, serial write-back), so 1M keys take 8 iterations.
constexpr int RS_SCAN_ITEMS = 16;
__global__ void __launch_bounds__(1024) rs_scan(uint32_t* data, int len) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < len; base += 1024 * RS_SCAN_ITEMS) {
        const int i0 = base + threadIdx.x * RS_SCAN_ITEMS;
        uint32_t item[RS_SCAN_ITEMS];
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < RS_SCAN_ITEMS; ++k) {
            item[k] = (i0 + k < len) ? data[i0 + k] : 0u;
            v += item[k];
        }
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = warp_sums[threadIdx.x], z = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, z, o);
                if (threadIdx.x >= o) z += y;
            }
            warp_sums[threadIdx.x] = z - w;  // exclusive prefix of the warp totals
        }
        __syncthreads();
        uint32_t run = x - v + warp_sums[threadIdx.x >> 5] + carry;
#pragma unroll
        for (int k = 0; k < RS_SCAN_ITEMS; ++k) {
            if (i0 + k < len) data[i0 + k] = run;
            run += item[k];
        }
        __syncthreads();
        if (threadIdx.x == 1023) carry = run;
        __syncthreads();
    }
}

// stable scatter of one tile.  Warp w owns the contiguous sub-tile [w*256, (w+1)*256) and walks it in 8 rounds of
// 32 consecutive keys, so (warp, round, lane) order == input order; ranks come from match_any + popc.
// FUSED = the (digit, block) offsets are computed here from the raw per-block histograms instead of by a separate rs_scan launch:
// offset(d, blk) = sum of all counters of the digits below d + the counters of digit d in the blocks before blk.  Every block redoes the
// 256 x nblocks row sums (L2-resident, 49 KB at 100k keys), which is cheaper than a single-block scan kernel and its launch gap as
// long as nblocks is small; the host keeps the scan kernel above RS_FUSE_MAX_BLOCKS.
constexpr int RS_FUSE_MAX_BLOCKS = 128;
template <class K, bool FUSED>
__global__ void __launch_bounds__(RS_THREADS) rs_scatter(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, int n, int shift,
                                                         const uint32_t* __restrict__ offsets, int nblocks, K* __restrict__ keys_out,
                                                         uint32_t* __restrict__ vals_out) {
    __shared__ uint32_t wcnt[RS_WARPS][256];
    __shared__ uint32_t digit_base[256];
    __shared__ uint32_t scan_warp[8];
    if (FUSED) {
        // thread d: total of digit d over all blocks, and the part of it that belongs to earlier blocks
        const int d = threadIdx.x;
        uint32_t total = 0, before_blk = 0;
        const uint32_t* row = offsets + size_t(d) * nblocks;
        for (int b = 0; b < nblocks; ++b) {
            const uint32_t c = row[b];
            total += c;
            if (b < int(blockIdx.x)) before_blk += c;
        }
        // exclusive scan of the 256 totals (8 warps)
        uint32_t x = total;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) scan_warp[threadIdx.x >> 5] = x;
        __syncthreads();
        uint32_t warp_before = 0;
        for (int w = 0; w < (threadIdx.x >> 5); ++w) warp_before += scan_warp[w];
        digit_base[d] = (x - total) + warp_before + before_blk;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int d = threadIdx.x; d < RS_WARPS * 256; d += RS_THREADS) (&wcnt[0][0])[d] = 0;
    __syncthreads();
    const int base = blockIdx.x * RS_TILE + warp * (32 * RS_ROUNDS);
    K key[RS_ROUNDS];
    uint32_t val[RS_ROUNDS], rank[RS_ROUNDS];
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        int i = base + r * 32 + lane;
        bool ok = i < n;
        key[r] = ok ? keys_in[i] : K(0);
        val[r] = ok ? vals_in[i] : 0u;
        uint32_t digit = uint32_t(key[r] >> shift) & 0xff;
        uint32_t active = __ballot_sync(0xffffffffu, ok);
        uint32_t same = __match_any_sync(0xffffffffu, ok ? digit : 0x100u + lane) & active;
        uint32_t before = __popc(same & ((1u << lane) - 1u));
        uint32_t prev = ok ? wcnt[warp][digit] : 0u;
        rank[r] = prev + before;
        __syncwarp();
        if (ok && before == 0) wcnt[warp][digit] = prev + __popc(same);  // leader of each digit group
        __syncwarp();
    }
    __syncthreads();
    // per digit (one thread each): exclusive prefix across the 8 warps + global offset of (digit, block)
    {
        const int d = threadIdx.x;
        uint32_t run = FUSED ? digit_base[d] : offsets[d * nblocks + blockIdx.x];
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) {
            uint32_t c = wcnt[w][d];
            wcnt[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        int i = base + r * 32 + lane;
        if (i < n) {
            uint32_t digit = uint32_t(key[r] >> shift) & 0xff;
            uint32_t pos = wcnt[warp][digit] + rank[r];
            keys_out[pos] = key[r];
            vals_out[pos] = val[r];
        }
    }
}

// exclusive scan of n 32-bit counts into 64-bit offsets (offsets[n] = total), three small launches:
// per-block sums (1024 counts each) -> single-block scan of the <= 1024 block sums -> per-block local scan + base.
__device__ __forceinline__ uint64_t block_exclusive_scan_1024(uint64_t v, uint64_t* warp_sums, uint64_t& block_total) {
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint64_t w = warp_sums[threadIdx.x], z = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, z, o);
            if (threadIdx.x >= o) z += y;
        }
        warp_sums[threadIdx.x] = z - w;
        if (threadIdx.x == 31) warp_sums[32] = z;
    }
    __syncthreads();
    block_total = warp_sums[32];
    return x - v + warp_sums[threadIdx.x >> 5];
}
__global__ void __launch_bounds__(1024) scan_block_sums(const uint32_t* __restrict__ counts, int n, uint64_t* __restrict__ block_sums) {
    __shared__ uint64_t ws[33];
    int i = blockIdx.x * 1024 + threadIdx.x;
    uint64_t total;
    block_exclusive_scan_1024(i < n ? counts[i] : 0u, ws, total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(1024) scan_block_offsets(uint64_t* __restrict__ block_sums, int nblocks, uint64_t* __restrict__ total_out) {
    __shared__ uint64_t ws[33];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        int i = base + threadIdx.x;
        uint64_t v = i < nblocks ? block_sums[i] : 0ull, total;
        uint64_t excl = block_exclusive_scan_1024(v, ws, total) + carry;
        if (i < nblocks) block_sums[i] = excl;
        __syncthreads();
        if (threadIdx.x == 0) carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = carry;
}
__global__ void __launch_bounds__(1024) scan_apply(const uint32_t* __restrict__ counts, int n, const uint64_t* __restrict__ block_offsets,
                                                   uint64_t* __restrict__ offsets) {
    __shared__ uint64_t ws[33];
    int i = blockIdx.x * 1024 + threadIdx.x;
    uint64_t total;
    uint64_t excl = block_exclusive_scan_1024(i < n ? counts[i] : 0u, ws, total);
    if (i < n) offsets[i] = excl + block_offsets[blockIdx.x];
}

__device__ __forceinline__ uint64_t hash64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}
__global__ void hash_insert(const uint64_t* __restrict__ keys, uint64_t n, uint64_t* table, uint64_t mask) {
    uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    uint64_t k = keys[i] + 1;  // 0 is the empty marker
    uint64_t h = hash64(k) & mask;
    for (;;) {
        unsigned long long prev = atomicCAS((unsigned long long*)&table[h], 0ull, (unsigned long long)k);
        if (prev == 0ull || prev == k) return;
        h = (h + 1) & mask;
    }
}
__device__ __forceinline__ bool hash_contains(const uint64_t* table, uint64_t mask, uint64_t key) {
    uint64_t k = key + 1;
    uint64_t h = hash64(k) & mask;
    for (;;) {
        uint64_t v = table[h];
        if (v == k) return true;
        if (v == 0) return false;
        h = (h + 1) & mask;
    }
}

}  // namespace
}  // namespace avn
