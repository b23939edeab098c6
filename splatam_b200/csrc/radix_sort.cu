// radix_sort.cu -- hand-written stable LSD radix sort of (u32 key, u32 value) pairs, 8-bit digits, three kernels per
// digit pass (reduce-then-scan), for sm_90a.
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
// A pass over sort tiles of 256 threads x 16 keys (4096 keys; 2048 up to 64K pairs):
//   1. upsweep: one CTA per tile counts the tile's digits (shared-memory atomics into one histogram per warp) and
//      writes counts[digit][tile], every entry of a live tile, so nothing is zeroed;
//   2. scan: one CTA per digit turns its row into the exclusive prefix over the tiles and writes the digit's total;
//   3. downsweep: one CTA per tile ranks its keys stably (warp-striped coalesced loads; per-warp ranking: the lanes
//      holding the same digit find each other by one ballot per digit bit, the lowest lane bumps the warp's bin
//      counter in shared memory), scatters keys and values into their tile-local sorted order in shared memory and
//      writes them to global memory in runs (one run per digit), so the global writes are coalesced.  A digit's
//      global base is the exclusive prefix of the digit totals plus its scanned count for this tile.
// No CTA waits on another, so a pass is deterministic and does not depend on the order CTAs are scheduled in.  The
// single-kernel pass with decoupled look-back that this replaces made every tile wait on a chain of predecessor tiles'
// status words (DESIGN.md section 5).
// Grids are sized by the capacity; every kernel derives the live tile count from n (a device-side count allowed).
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

struct RadixTemp {
    uint32_t* totals;    // [kBins] keys per digit
    uint32_t* counts;    // [kBins][stride]: per-tile digit counts, scanned in place into per-tile digit bases
    uint32_t* pk;        // ping-pong keys   [capacity]
    uint32_t* pv;        // ping-pong values [capacity]
    size_t bytes;
    int tiles, stride;
};

inline int tile_items_for(int capacity) { return kSortThreads * (capacity <= kSmallSortLimit ? kItemsSmall : kItemsLarge); }

RadixTemp radix_layout(void* temp, int capacity) {
    RadixTemp t;
    Carver c(temp);
    const int kTileItems = tile_items_for(capacity);
    t.tiles = (capacity + kTileItems - 1) / kTileItems;
    // Past kSmallSortLimit the tiles double in size, so the tiles in use halve.  Reserve count columns up to the
    // small-tile count at the limit, so the temp size never decreases as the capacity grows and a temp sized for one
    // capacity serves every smaller one.
    const int reserve_tiles = capacity > kSmallSortLimit ? kSmallSortLimit / (kSortThreads * kItemsSmall) : 1;
    t.stride = ((t.tiles > reserve_tiles ? t.tiles : reserve_tiles) + 3) & ~3;   // 16-B aligned rows
    t.totals = c.take<uint32_t>(kBins);
    t.counts = c.take<uint32_t>((size_t)kBins * (size_t)t.stride);
    t.pk = c.take<uint32_t>((size_t)(capacity > 0 ? capacity : 1));
    t.pv = c.take<uint32_t>((size_t)(capacity > 0 ? capacity : 1));
    t.bytes = c.used();
    return t;
}

__device__ __forceinline__ int live_count(int capacity, const int32_t* n_dev) {
    return n_dev ? min(*n_dev, capacity) : capacity;
}

// The lanes of the warp holding the same digit d (mask = the digit's bits): one ballot per digit bit.  The hardware
// match instruction (__match_any_sync) costs more the more distinct values a warp holds; on random 8-bit digits it
// made the ranking the longest part of a pass (DESIGN.md section 5).
__device__ __forceinline__ uint32_t match_digit(uint32_t d, uint32_t mask) {
    uint32_t peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        if (!((mask >> b) & 1u)) break;   // mask is 2^width - 1, the same in every lane
        const bool set = (d >> b) & 1u;
        const uint32_t bal = __ballot_sync(0xffffffffu, set);
        peers &= set ? bal : ~bal;
    }
    return peers;
}

template <int kItems>
__global__ void __launch_bounds__(kSortThreads)
radix_upsweep_kernel(const uint32_t* __restrict__ keys_in, int capacity, const int32_t* __restrict__ n_dev, int shift,
                     uint32_t mask, int stride, uint32_t* __restrict__ counts) {
    constexpr int kTileItems = kSortThreads * kItems;
    __shared__ uint32_t s_hist[kSortWarps][kBins];
    const int tid = threadIdx.x;
    const int n = live_count(capacity, n_dev);
    const long long tile_base = (long long)blockIdx.x * kTileItems;
    if (tile_base >= n) return;
    const int valid = (int)min((long long)kTileItems, (long long)n - tile_base);
    for (int i = tid; i < kSortWarps * kBins; i += kSortThreads) (&s_hist[0][0])[i] = 0u;
    __syncthreads();
    uint32_t k[kItems];
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int li = j * kSortThreads + tid;
        k[j] = li < valid ? __ldg(keys_in + tile_base + li) : 0u;
    }
    uint32_t* const h = s_hist[tid >> 5];   // one histogram per warp: only lanes of one warp contend for a bin
#pragma unroll
    for (int j = 0; j < kItems; ++j)
        if (j * kSortThreads + tid < valid) atomicAdd(&h[(k[j] >> shift) & mask], 1u);
    __syncthreads();
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) c += s_hist[w][tid];
    counts[(size_t)tid * stride + blockIdx.x] = c;
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

// Row d = blockIdx.x of counts (the live tiles' counts of digit d) -> its exclusive prefix; totals[d] = the row's sum.
// Each thread takes 4 consecutive tiles per round (one 16-B load: rows start 16-B aligned), 1024 tiles per round.
__global__ void __launch_bounds__(kSortThreads)
radix_scan_kernel(int capacity, const int32_t* __restrict__ n_dev, int tile_items, int stride,
                  uint32_t* __restrict__ counts, uint32_t* __restrict__ totals) {
    __shared__ uint32_t s_scan[kSortWarps];
    const int tid = threadIdx.x;
    const int n = live_count(capacity, n_dev);
    const int tiles = n > 0 ? (int)(((long long)n + tile_items - 1) / tile_items) : 0;
    uint32_t* const row = counts + (size_t)blockIdx.x * stride;
    uint32_t carry = 0;
    for (int t0 = 0; t0 < tiles; t0 += 4 * kSortThreads) {
        const int first = t0 + 4 * tid;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (first < tiles) {   // first + 3 < stride: the stride is a multiple of 4
            v = *reinterpret_cast<const uint4*>(row + first);
            if (first + 1 >= tiles) v.y = 0u;
            if (first + 2 >= tiles) v.z = 0u;
            if (first + 3 >= tiles) v.w = 0u;
        }
        const uint32_t sum = v.x + v.y + v.z + v.w;
        const uint32_t excl = carry + block_exclusive_scan(sum, s_scan);
        if (first < tiles) row[first] = excl;
        if (first + 1 < tiles) row[first + 1] = excl + v.x;
        if (first + 2 < tiles) row[first + 2] = excl + v.x + v.y;
        if (first + 3 < tiles) row[first + 3] = excl + v.x + v.y + v.z;
        if (tid == kSortThreads - 1) s_scan[0] = excl + sum;
        __syncthreads();
        carry = s_scan[0];
        __syncthreads();
    }
    if (tid == 0) totals[blockIdx.x] = carry;
}

template <bool IOTA, int kItems>
__global__ void __launch_bounds__(kSortThreads)
radix_downsweep_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                       uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int capacity,
                       const int32_t* __restrict__ n_dev, int shift, uint32_t mask, int stride,
                       const uint32_t* __restrict__ counts, const uint32_t* __restrict__ totals) {
    constexpr int kTileItems = kSortThreads * kItems;
    __shared__ uint32_t s_keys[kTileItems];
    __shared__ uint32_t s_vals[kTileItems];
    __shared__ uint32_t s_whist[kSortWarps][kBins];
    __shared__ uint32_t s_tile_excl[kBins];
    __shared__ uint32_t s_gbase[kBins];
    __shared__ uint32_t s_scan[kSortWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = live_count(capacity, n_dev);
    const long long tile_base = (long long)blockIdx.x * kTileItems;
    if (tile_base >= n) return;
    const int valid = (int)min((long long)kTileItems, (long long)n - tile_base);
    // this tile's base of digit tid among the keys of that digit, and the digit's total (both from the scan)
    const uint32_t digit_base = __ldg(counts + (size_t)tid * stride + blockIdx.x);
    const uint32_t digit_total = __ldg(totals + tid);
    for (int i = tid; i < kSortWarps * kBins; i += kSortThreads) (&s_whist[0][0])[i] = 0u;
    __syncthreads();

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
        const uint32_t peers = match_digit(d, mask);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == leader) { base = whist[d]; whist[d] = base + __popc(peers); }
        base = __shfl_sync(0xffffffffu, base, leader);
        rank[j] = base + __popc(peers & lt);
        __syncwarp();
    }
    __syncthreads();

    // 2. per digit (thread d): exclusive prefix over the warps, tile total; global base of the digit in this tile
    uint32_t count = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) { const uint32_t c = s_whist[w][tid]; s_whist[w][tid] = count; count += c; }
    const uint32_t tile_excl = block_exclusive_scan(count, s_scan);
    const uint32_t digit_excl = block_exclusive_scan(digit_total, s_scan);
    s_tile_excl[tid] = tile_excl;
    s_gbase[tid] = digit_excl + digit_base - tile_excl;   // global position = s_gbase[digit] + tile-local position
    __syncthreads();

    // 3. tile-local scatter in shared memory, then run-wise coalesced global writes
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
    (void)bits;   // the count matrix is re-used by every pass
    return radix_layout(nullptr, capacity).bytes;
}

int radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out,
                     int capacity, const int32_t* n_dev, int begin_bit, int end_bit, void* temp, size_t temp_bytes,
                     cudaStream_t st) {
    if (capacity <= 0) return SB_OK;
    const int passes = (end_bit - begin_bit + 7) / 8;
    if (passes < 1 || passes > kMaxPasses || begin_bit < 0 || end_bit > 32 || capacity >= (1 << 30) || !temp)
        return SB_ERR_BAD_ARG;
    RadixTemp t = radix_layout(temp, capacity);
    if (temp_bytes < t.bytes) return SB_ERR_WORKSPACE;
    const bool small = capacity <= kSmallSortLimit;
    const uint32_t* src_k = keys_in;
    const uint32_t* src_v = vals_in;
    for (int p = 0; p < passes; ++p) {
        // destinations alternate so that the LAST pass lands in (keys_out, vals_out)
        const bool to_out = ((passes - 1 - p) & 1) == 0;
        uint32_t* dst_k = to_out ? keys_out : t.pk;
        uint32_t* dst_v = to_out ? vals_out : t.pv;
        const int lo = begin_bit + 8 * p, width = min(8, end_bit - lo);
        const uint32_t mask = (1u << width) - 1u;
        if (small) radix_upsweep_kernel<kItemsSmall><<<t.tiles, kSortThreads, 0, st>>>(src_k, capacity, n_dev, lo, mask, t.stride, t.counts);
        else radix_upsweep_kernel<kItemsLarge><<<t.tiles, kSortThreads, 0, st>>>(src_k, capacity, n_dev, lo, mask, t.stride, t.counts);
        SB_LAUNCH_CHECK("radix_upsweep_kernel");
        radix_scan_kernel<<<kBins, kSortThreads, 0, st>>>(capacity, n_dev, tile_items_for(capacity), t.stride, t.counts,
                                                            t.totals);
        SB_LAUNCH_CHECK("radix_scan_kernel");
#define SB_SORT_PASS(IOTA, ITEMS)                                                                                   \
        radix_downsweep_kernel<IOTA, ITEMS><<<t.tiles, kSortThreads, 0, st>>>(src_k, IOTA ? nullptr : src_v, dst_k,    \
                                                                              dst_v, capacity, n_dev, lo, mask,         \
                                                                              t.stride, t.counts, t.totals)
        const bool iota = (p == 0 && vals_in == nullptr);
        if (iota && small) SB_SORT_PASS(true, kItemsSmall);
        else if (iota) SB_SORT_PASS(true, kItemsLarge);
        else if (small) SB_SORT_PASS(false, kItemsSmall);
        else SB_SORT_PASS(false, kItemsLarge);
#undef SB_SORT_PASS
        SB_LAUNCH_CHECK("radix_downsweep_kernel");
        src_k = dst_k;
        src_v = dst_v;
    }
    return SB_OK;
}

}  // namespace sb
