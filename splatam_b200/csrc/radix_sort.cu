// radix_sort.cu -- hand-written stable LSD radix sort of (u32 key, u32 value) pairs, 8-bit digits, one kernel per
// digit pass with decoupled look-back ("onesweep"), for sm_90a.
//
// Where the reference calls cub::DeviceRadixSort::SortPairs on 64-bit (tile | depth) keys over num_rendered pairs
// (X/cuda_rasterizer/rasterizer_impl.cu:304-309), this repo orders the P Gaussians by their 32 depth bits once
// (4 passes over P pairs) and then the R tile instances by tile id alone (2 passes over R pairs at 1200x680), see
// binning.cu.  Both orderings run through this file.  What the library sort could not give this pipeline:
//   * the pair count may live on the DEVICE (n_dev): the sync-free / CUDA-graph mode sorts exactly num_rendered
//     instances instead of the padded capacity, with no host read-back;
//   * the first pass can synthesise its payload (vals_in == nullptr -> the element's index), so no iota array is
//     written or read;
//   * the input keys are never modified (the depth keys are re-used by the blend and by the key export).
//
// Structure of a pass (one CTA = 256 threads x 16 keys = one 4096-key tile, tiles ticketed in launch order):
//   1. warp-striped coalesced key loads; per-warp stable ranking with __match_any_sync (all lanes holding the same
//      digit find each other, the lowest lane bumps the warp's bin counter in shared memory);
//   2. per digit: exclusive prefix over the 8 warps, tile total;
//   3. per digit (one thread each): decoupled look-back over the predecessor tiles' status words
//      {2-bit flag | 30-bit count}: publish AGGREGATE, sum predecessors until an INCLUSIVE one, publish INCLUSIVE;
//   4. keys and values are first scattered inside shared memory into their tile-local sorted order, then written
//      to global memory in runs (one run per digit), so the global writes are coalesced.
// A single up-front kernel builds the digit histograms of all passes (global bin bases).
#include "radix_sort.cuh"
#include "common.cuh"

namespace sb {

namespace {

constexpr int kBins = 256;
constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kItemsLarge = 16, kItemsSmall = 8;       // keys per thread: 4096- or 2048-key tiles
constexpr int kSmallSortLimit = 64 << 10;              // tiny inputs only: 2048-key tiles lose to 4096-key tiles at 1M keys
constexpr int kMaxPasses = 4;
constexpr uint32_t kFlagAgg = 1u << 30, kFlagInc = 2u << 30, kValMask = (1u << 30) - 1u;

struct RadixTemp {
    uint32_t* hist;      // [kMaxPasses][kBins]
    uint32_t* tickets;   // [64] (one per pass)
    uint32_t* status;    // [passes][tiles][kBins]
    uint32_t* pk;        // ping-pong keys   [capacity]
    uint32_t* pv;        // ping-pong values [capacity]
    size_t zero_bytes;   // hist + tickets + status are contiguous and zeroed per sort
    size_t bytes;
    int tiles;
};

inline int tile_items_for(int capacity) { return kSortThreads * (capacity <= kSmallSortLimit ? kItemsSmall : kItemsLarge); }

RadixTemp radix_layout(void* temp, int capacity, int passes) {
    RadixTemp t;
    Carver c(temp);
    const int kTileItems = tile_items_for(capacity);
    t.tiles = (capacity + kTileItems - 1) / kTileItems;
    t.hist = c.take<uint32_t>((size_t)kMaxPasses * kBins);
    t.tickets = c.take<uint32_t>(64);
    const int live_tiles = t.tiles > 0 ? t.tiles : 1;
    t.status = c.take<uint32_t>((size_t)passes * (size_t)live_tiles * kBins);
    t.zero_bytes = c.used();
    // Past kSmallSortLimit the tiles double in size, so the status words of the tiles in use halve.  Reserve (without
    // zeroing) up to the small-tile count at the limit, so the temp size never decreases as the capacity grows and a
    // temp sized for one capacity serves every smaller one.
    const int reserve_tiles = capacity > kSmallSortLimit ? kSmallSortLimit / (kSortThreads * kItemsSmall) : 0;
    if (reserve_tiles > live_tiles) c.take<uint32_t>((size_t)passes * (size_t)(reserve_tiles - live_tiles) * kBins);
    t.pk = c.take<uint32_t>((size_t)(capacity > 0 ? capacity : 1));
    t.pv = c.take<uint32_t>((size_t)(capacity > 0 ? capacity : 1));
    t.bytes = c.used();
    return t;
}

__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void __launch_bounds__(256)
radix_hist_kernel(const uint32_t* __restrict__ keys, int capacity, const int32_t* __restrict__ n_dev, int begin_bit,
                  int end_bit, int passes, uint32_t* __restrict__ hist) {
    __shared__ uint32_t sh[kMaxPasses][kBins];
    for (int i = threadIdx.x; i < kMaxPasses * kBins; i += blockDim.x) (&sh[0][0])[i] = 0u;
    __syncthreads();
    const int n = n_dev ? min(*n_dev, capacity) : capacity;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t key = __ldg(keys + i);
        for (int p = 0; p < passes; ++p) {
            const int lo = begin_bit + 8 * p, width = min(8, end_bit - lo);
            atomicAdd(&sh[p][(key >> lo) & ((1u << width) - 1u)], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < passes * kBins; i += blockDim.x) {
        const uint32_t v = (&sh[0][0])[i];
        if (v) atomicAdd(hist + i, v);
    }
}

// Exclusive prefix of one value per thread over the 256 threads of the CTA.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp /* [8] */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
        if (lane >= off) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t base = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) base += (w < warp) ? s_warp[w] : 0u;
    __syncthreads();
    return base + inc - v;
}

template <bool IOTA, int kItems>
__global__ void __launch_bounds__(kSortThreads)
radix_onesweep_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                      uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int capacity,
                      const int32_t* __restrict__ n_dev, int shift, uint32_t mask, const uint32_t* __restrict__ hist,
                      uint32_t* __restrict__ ticket, uint32_t* __restrict__ status) {
    constexpr int kTileItems = kSortThreads * kItems;
    __shared__ uint32_t s_keys[kTileItems];
    __shared__ uint32_t s_vals[kTileItems];
    __shared__ uint32_t s_whist[kSortWarps][kBins];
    __shared__ uint32_t s_tile_excl[kBins];
    __shared__ uint32_t s_gbase[kBins];
    __shared__ uint32_t s_scan[kSortWarps];
    __shared__ uint32_t s_tile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = n_dev ? min(*n_dev, capacity) : capacity;
    if (tid == 0) s_tile = atomicAdd(ticket, 1u);
    for (int i = tid; i < kSortWarps * kBins; i += kSortThreads) (&s_whist[0][0])[i] = 0u;
    __syncthreads();
    const uint32_t tile = s_tile;
    const long long tile_base = (long long)tile * kTileItems;
    if (tile_base >= n) return;                      // tickets beyond the live range (device-side n)
    const int valid = (int)min((long long)kTileItems, (long long)n - tile_base);

    // 1. load + rank.  Element order inside the tile is (warp, round, lane), i.e. the global index order.
    uint32_t keys[kItems];
    uint32_t rank[kItems];
    const int warp_base = warp * (kItems * 32);
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int li = warp_base + j * 32 + lane;
        keys[j] = li < valid ? __ldg(keys_in + tile_base + li) : 0xFFFFFFFFu;   // padding sorts to the tile's tail
    }
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t* const whist = s_whist[warp];
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const uint32_t d = (keys[j] >> shift) & mask;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == leader) { base = whist[d]; whist[d] = base + __popc(peers); }
        base = __shfl_sync(0xffffffffu, base, leader);
        rank[j] = base + __popc(peers & lt);
        __syncwarp();
    }
    __syncthreads();

    // 2. per digit (thread d): exclusive prefix over the warps, tile total
    uint32_t count = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) { const uint32_t c = s_whist[w][tid]; s_whist[w][tid] = count; count += c; }

    // 3. decoupled look-back: number of keys with this digit in all predecessor tiles
    uint32_t* const my = status + (size_t)tile * kBins + tid;
    uint32_t prev = 0;
    if (tile == 0) {
        st_relaxed(my, kFlagInc | count);
    } else {
        st_relaxed(my, kFlagAgg | count);
        // walk back over the predecessors, kLook status words in flight at a time (the loads are independent, so their
        // L2 latencies overlap; a strictly serial walk costs one round trip per predecessor tile)
        constexpr int kLook = 8;
        long long t = (long long)tile - 1;
        bool done = false;
        while (t >= 0 && !done) {
            const int nb = (int)min((long long)kLook, t + 1);
            uint32_t sw[kLook];
#pragma unroll
            for (int i = 0; i < kLook; ++i)
                sw[i] = i < nb ? ld_relaxed(status + (size_t)(t - i) * kBins + tid) : 0u;
#pragma unroll
            for (int i = 0; i < kLook; ++i) {
                if (i < nb && !done) {
                    uint32_t sv = sw[i];
                    while ((sv >> 30) == 0u) sv = ld_relaxed(status + (size_t)(t - i) * kBins + tid);
                    prev += sv & kValMask;
                    done = (sv >> 30) == 2u;
                }
            }
            t -= nb;
        }
        st_relaxed(my, kFlagInc | (prev + count));
    }
    const uint32_t tile_excl = block_exclusive_scan(count, s_scan);
    const uint32_t hist_excl = block_exclusive_scan(__ldg(hist + tid), s_scan);
    s_tile_excl[tid] = tile_excl;
    s_gbase[tid] = hist_excl + prev - tile_excl;     // global position = s_gbase[digit] + tile-local position
    __syncthreads();

    // 4. tile-local scatter in shared memory, then run-wise coalesced global writes
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const uint32_t d = (keys[j] >> shift) & mask;
        const uint32_t pos = s_tile_excl[d] + whist[d] + rank[j];
        const int li = warp_base + j * 32 + lane;
        s_keys[pos] = keys[j];
        s_vals[pos] = IOTA ? (uint32_t)(tile_base + li) : (li < valid ? __ldg(vals_in + tile_base + li) : 0u);
    }
    __syncthreads();
    for (int i = tid; i < valid; i += kSortThreads) {
        const uint32_t k = s_keys[i];
        const uint32_t pos = s_gbase[(k >> shift) & mask] + (uint32_t)i;
        keys_out[pos] = k;
        vals_out[pos] = s_vals[i];
    }
}

}  // namespace

size_t radix_temp_bytes(int capacity, int bits) {
    const int passes = (bits + 7) / 8;
    return radix_layout(nullptr, capacity, passes < 1 ? 1 : passes).bytes;
}

int radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out,
                     int capacity, const int32_t* n_dev, int begin_bit, int end_bit, void* temp, size_t temp_bytes,
                     cudaStream_t st) {
    if (capacity <= 0) return SB_OK;
    const int passes = (end_bit - begin_bit + 7) / 8;
    if (passes < 1 || passes > kMaxPasses || begin_bit < 0 || end_bit > 32 || capacity >= (1 << 30) || !temp)
        return SB_ERR_BAD_ARG;
    RadixTemp t = radix_layout(temp, capacity, passes);
    if (temp_bytes < t.bytes) return SB_ERR_WORKSPACE;
    SB_CUDA_CHECK(cudaMemsetAsync(temp, 0, t.zero_bytes, st));
    const int hist_blocks = min((capacity + 4 * 256 - 1) / (4 * 256), 132 * 8);   // 132 SMs x 8
    radix_hist_kernel<<<hist_blocks, 256, 0, st>>>(keys_in, capacity, n_dev, begin_bit, end_bit, passes, t.hist);
    SB_LAUNCH_CHECK("radix_hist_kernel");
    const uint32_t* src_k = keys_in;
    const uint32_t* src_v = vals_in;
    for (int p = 0; p < passes; ++p) {
        // destinations alternate so that the LAST pass lands in (keys_out, vals_out)
        const bool to_out = ((passes - 1 - p) & 1) == 0;
        uint32_t* dst_k = to_out ? keys_out : t.pk;
        uint32_t* dst_v = to_out ? vals_out : t.pv;
        const int lo = begin_bit + 8 * p, width = min(8, end_bit - lo);
        const uint32_t mask = (1u << width) - 1u;
        uint32_t* status = t.status + (size_t)p * (size_t)t.tiles * kBins;
#define SB_SORT_PASS(IOTA, ITEMS)                                                                                   \
        radix_onesweep_kernel<IOTA, ITEMS><<<t.tiles, kSortThreads, 0, st>>>(src_k, IOTA ? nullptr : src_v, dst_k, dst_v,  \
                                                                             capacity, n_dev, lo, mask, t.hist + p * kBins, \
                                                                             t.tickets + p, status)
        const bool iota = (p == 0 && vals_in == nullptr), small = capacity <= kSmallSortLimit;
        if (iota && small) SB_SORT_PASS(true, kItemsSmall);
        else if (iota) SB_SORT_PASS(true, kItemsLarge);
        else if (small) SB_SORT_PASS(false, kItemsSmall);
        else SB_SORT_PASS(false, kItemsLarge);
#undef SB_SORT_PASS
        SB_LAUNCH_CHECK("radix_onesweep_kernel");
        src_k = dst_k;
        src_v = dst_v;
    }
    return SB_OK;
}

}  // namespace sb
