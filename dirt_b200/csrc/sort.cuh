// sort.cuh -- the stable LSD radix sort of (key, id) pairs of the deterministic backward passes (DESIGN.md §7.5): the
// texture lookups by base texel (texture.cu) and the shadow-map lookups by base texel (shadow.cu, §7.15).
//
// 8 bits per pass, and only as many passes as the largest key, the sentinel, needs.  The first pass computes the keys
// with the caller's Key (key(i) for element i; an element that adds nothing gets the sentinel) and takes the ids from
// the positions.  Per pass: a histogram per tile of RS_TILE elements, an exclusive scan of each digit's row of the
// [digit][tile] count matrix (one CTA per digit), and a scatter in which an element's rank in its tile comes from
// MATCH.ANY on the digit and the warps' digit counts taken in warp order.  The output is unique.  Then
// tex_segment_bounds_kernel: offsets[k] = the first sorted position whose key is >= k, so that the elements of key x
// are the segment [offsets[x], offsets[x + 1]).
#pragma once

namespace dirt {

namespace {

constexpr int RS_THREADS = 256;             // sort CTA: one thread per digit value
constexpr int RS_RADIX = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_TILE = 4096;               // elements per sort tile, 16 per thread

// Exclusive scan of one value per thread over the RS_THREADS threads of the CTA; *total gets the sum.  Contains
// __syncthreads(); warp_sums is RS_WARPS words of shared memory.
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned* warp_sums, unsigned* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    unsigned before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) {
        const unsigned s = warp_sums[w];
        before += w < warp ? s : 0u;
        all += s;
    }
    __syncthreads();
    *total = all;
    return before + x - v;
}

// counts[digit][tile]: how many lookups of the tile have the digit (key >> shift) & 255
template <bool FIRST, class Key>
__global__ void __launch_bounds__(RS_THREADS) tex_sort_hist_kernel(const unsigned* __restrict__ keys, Key key, long long n,
                                                                   int shift, unsigned* __restrict__ counts, int tiles)
{
    __shared__ unsigned hist[RS_RADIX];
    hist[threadIdx.x] = 0;
    __syncthreads();
    const long long first = (long long)blockIdx.x * RS_TILE;
    for (int j = 0; j < RS_TILE / RS_THREADS; ++j) {
        const long long i = first + j * RS_THREADS + threadIdx.x;
        if (i < n) {
            const unsigned k = FIRST ? key(i) : __ldg(keys + i);
            atomicAdd(&hist[(k >> shift) & 255u], 1u);
        }
    }
    __syncthreads();
    counts[(size_t)threadIdx.x * tiles + blockIdx.x] = hist[threadIdx.x];
}

// one CTA per digit: its row of tile counts becomes the exclusive prefix, in place; the row's sum goes to digit_total
__global__ void __launch_bounds__(RS_THREADS) tex_sort_scan_kernel(unsigned* __restrict__ counts,
                                                                   unsigned* __restrict__ digit_total, int tiles)
{
    __shared__ unsigned warp_sums[RS_WARPS];
    unsigned* row = counts + (size_t)blockIdx.x * tiles;
    unsigned carry = 0;
    for (int base = 0; base < tiles; base += RS_THREADS) {
        const int i = base + threadIdx.x;
        const unsigned v = i < tiles ? row[i] : 0u;
        unsigned total;
        const unsigned ex = block_exclusive_scan(v, warp_sums, &total);
        if (i < tiles) row[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) digit_total[blockIdx.x] = carry;
}

// Stable scatter of one tile.  Its lookups go in 16 rounds of RS_THREADS consecutive ones; in a round a lookup's slot is
// the tile's running slot of its digit, plus the lookups of the lower warps with that digit, plus its rank among its
// warp's lanes with that digit.  Thread dgt keeps the running slot of digit dgt.
template <bool FIRST, class Key>
__global__ void __launch_bounds__(RS_THREADS) tex_sort_scatter_kernel(const unsigned* __restrict__ keys_in,
                                                                      const int* __restrict__ ids_in, Key key_of,
                                                                      long long n, int shift,
                                                                      const unsigned* __restrict__ counts,
                                                                      const unsigned* __restrict__ digit_total, int tiles,
                                                                      unsigned* __restrict__ keys_out,
                                                                      int* __restrict__ ids_out)
{
    __shared__ unsigned warp_sums[RS_WARPS];
    __shared__ unsigned wcount[RS_WARPS][RS_RADIX];
    __shared__ unsigned woff[RS_WARPS][RS_RADIX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, dgt = threadIdx.x;
    unsigned all;
    // the lookups of the smaller digits, then those of digit dgt in the earlier tiles
    unsigned run = block_exclusive_scan(digit_total[dgt], warp_sums, &all) + counts[(size_t)dgt * tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) wcount[w][dgt] = 0;
    __syncthreads();
    const long long first = (long long)blockIdx.x * RS_TILE;
    for (int j = 0; j < RS_TILE / RS_THREADS; ++j) {
        const long long i = first + j * RS_THREADS + threadIdx.x;
        const bool live = i < n;
        unsigned key = 0;
        int id = 0;
        if (live) {
            key = FIRST ? key_of(i) : __ldg(keys_in + i);
            id = FIRST ? (int)i : __ldg(ids_in + i);
        }
        const unsigned digit = live ? (key >> shift) & 255u : (unsigned)RS_RADIX;
        const unsigned peers = __match_any_sync(0xffffffffu, digit);
        const unsigned rank = __popc(peers & ((1u << lane) - 1u));
        if (live && rank == 0) wcount[warp][digit] = __popc(peers);
        __syncthreads();
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) {
            woff[w][dgt] = run;
            run += wcount[w][dgt];
            wcount[w][dgt] = 0;
        }
        __syncthreads();
        if (live) {
            const unsigned pos = woff[warp][digit] + rank;
            keys_out[pos] = key;
            ids_out[pos] = id;
        }
    }
}

// offsets[k] = the first position of the sorted keys that is >= k, k = 0 .. sentinel + 1
__global__ void __launch_bounds__(RS_THREADS) tex_segment_bounds_kernel(const unsigned* __restrict__ keys, long long n,
                                                                         unsigned sentinel, int* __restrict__ offsets)
{
    const long long stride = (long long)gridDim.x * RS_THREADS;
    for (long long k = (long long)blockIdx.x * RS_THREADS + threadIdx.x; k <= (long long)sentinel + 1; k += stride) {
        long long lo = 0, hi = n;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(keys + mid) < (unsigned)k) lo = mid + 1;
            else hi = mid;
        }
        offsets[k] = (int)lo;
    }
}

// sort passes: one per 8 bits of the largest key, the sentinel
inline int sort_passes(unsigned sentinel)
{
    int bits = 0;
    while (bits < 32 && (sentinel >> bits) != 0) ++bits;
    return (bits + 7) / 8;
}

// Sorts the n elements' (key, id) pairs: keys[2], ids[2] are the ping-pong buffers of n entries each, counts
// RS_RADIX * ceil(n / RS_TILE) and digit_total RS_RADIX words of scratch.  The sorted pairs end in keys[*last],
// ids[*last].  n > 0.
template <class Key>
cudaError_t sort_by_key(const Key& key, long long n, unsigned sentinel, unsigned* const keys[2], int* const ids[2],
                        unsigned* counts, unsigned* digit_total, cudaStream_t stream, int* last)
{
    cudaError_t e;
    const int tiles = (int)((n + RS_TILE - 1) / RS_TILE), passes = sort_passes(sentinel);
    for (int p = 0; p < passes; ++p) {
        const unsigned* kin = keys[(p + 1) & 1];
        const int* iin = ids[(p + 1) & 1];
        unsigned* kout = keys[p & 1];
        int* iout = ids[p & 1];
        if (p == 0) tex_sort_hist_kernel<true><<<tiles, RS_THREADS, 0, stream>>>(kin, key, n, 0, counts, tiles);
        else tex_sort_hist_kernel<false><<<tiles, RS_THREADS, 0, stream>>>(kin, key, n, 8 * p, counts, tiles);
        if ((e = launched()) != cudaSuccess) return e;
        tex_sort_scan_kernel<<<RS_RADIX, RS_THREADS, 0, stream>>>(counts, digit_total, tiles);
        if ((e = launched()) != cudaSuccess) return e;
        if (p == 0)
            tex_sort_scatter_kernel<true><<<tiles, RS_THREADS, 0, stream>>>(kin, iin, key, n, 0, counts, digit_total, tiles,
                                                                             kout, iout);
        else
            tex_sort_scatter_kernel<false><<<tiles, RS_THREADS, 0, stream>>>(kin, iin, key, n, 8 * p, counts, digit_total,
                                                                              tiles, kout, iout);
        if ((e = launched()) != cudaSuccess) return e;
    }
    *last = (passes - 1) & 1;
    return cudaSuccess;
}

}  // namespace

}  // namespace dirt
