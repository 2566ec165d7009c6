// radix_sort.cuh - single-sweep ("onesweep") stable LSD radix sort for sm_90a.
//
// Replaces cub::DeviceRadixSort::SortPairs / cub::DeviceScan::InclusiveSum at
// DGR/cuda_rasterizer/rasterizer_impl.cu:278,304-309.  Hand-written: one global
// histogram kernel for all digit passes, then ONE kernel per 8-bit digit that
// ranks its 4096-item tile with warp match-any multisplit, publishes its digit
// counts in a decoupled look-back chain and scatters through shared memory so
// the global writes are digit-contiguous runs.
//
// Stability: a block's items are consumed in global index order
// (warp-striped: warp w owns [w*512, w*512+512), item i of lane l is i*32+l),
// ranks inside a warp follow (i, lane) order, warps are prefixed in order, and
// blocks are chained in ticket order == index order.
#pragma once
#include "common.cuh"

namespace s3g {

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_volatile_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

constexpr uint32_t LB_FLAG_AGG = 1u << 30;
constexpr uint32_t LB_FLAG_INCL = 2u << 30;
constexpr uint32_t LB_VALUE_MASK = (1u << 30) - 1u;
constexpr int LB_WINDOW = 8;

// block-wide exclusive scan of one value per thread (256 threads)
__device__ __forceinline__ uint32_t block_excl_scan_256(uint32_t v, uint32_t* s_warp /*[8]*/,
                                                        uint32_t* total = nullptr) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t wbase = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < SORT_THREADS / 32; ++w) {
        uint32_t c = s_warp[w];
        if (w < warp) wbase += c;
        tot += c;
    }
    if (total) *total = tot;
    __syncthreads();
    return wbase + inc - v;
}

// The sort kernels and their host driver are compiled in their own translation unit (radix_sort.cu,
// which defines S3G_RADIX_SORT_IMPL); everyone else sees the declaration only.
// n: item count known on the host, or the capacity when `n_dev` (device word with the true count, clamped to n)
// is given.  prepared: the caller already zeroed the temp block (radix_sort_prepare, e.g. folded into a larger
// memset).  hist_ready (implies prepared): a producer kernel already wrote the digit histograms
// st.hist[pass][digit]; otherwise the driver runs sort_histogram_kernel.  keys_spare: a second key scratch of n
// items; the intermediate keys then alternate between keys_tmp and keys_spare and keys_in keeps the input keys
// (without it the second pass writes its keys back into keys_in).
cudaError_t radix_sort_prepare(const SortTemp& st, cudaStream_t stream);
cudaError_t radix_sort_pairs(uint32_t n, uint32_t* keys_in, uint32_t* vals_in, uint32_t* keys_tmp,
                             uint32_t* vals_tmp, uint32_t* keys_final, uint32_t* vals_final, int begin_bit,
                             int end_bit, const SortTemp& st, cudaStream_t stream,
                             const uint32_t* n_dev = nullptr, bool hist_ready = false, bool prepared = false,
                             uint32_t* keys_spare = nullptr);

#ifdef S3G_RADIX_SORT_IMPL
// ---- histogram of every digit of every pass in one read of the keys -------
// grid: any (grid-stride by tiles of 256*16); hist: [npass][RADIX], pre-zeroed.
__global__ void __launch_bounds__(SORT_THREADS)
sort_histogram_kernel(const uint32_t* __restrict__ keys, uint32_t n, int begin_bit, int end_bit,
                      int npass, uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_hist[SORT_MAX_PASSES][RADIX];
    for (int i = threadIdx.x; i < SORT_MAX_PASSES * RADIX; i += SORT_THREADS)
        (&s_hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t stride = gridDim.x * SORT_THREADS;
    for (uint32_t i = blockIdx.x * SORT_THREADS + threadIdx.x; i < n; i += stride) {
        uint32_t k = keys[i];
#pragma unroll
        for (int p = 0; p < SORT_MAX_PASSES; ++p) {
            if (p < npass) {
                int shift = begin_bit + p * RADIX_BITS;
                int bits = min(RADIX_BITS, end_bit - shift);
                uint32_t d = (k >> shift) & ((1u << bits) - 1u);
                atomicAdd(&s_hist[p][d], 1u);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < npass * RADIX; i += SORT_THREADS) {
        uint32_t c = (&s_hist[0][0])[i];
        if (c) atomicAdd(&hist[i], c);
    }
}


// ---- one digit pass --------------------------------------------------------
// grid: exactly ceil(n / SORT_TILE) blocks.  status: [nblk][RADIX] zeroed.
// Block order = data order must be START order (a block only waits on blocks that are running), so positions are
// handed out by a ticket atomic.  Alternatives: blockIdx order (no ticket) would avoid the same-address atomics
// that serialise in L2 at the start of every pass, but relies on in-order dispatch, so it is not used; one ticket per
// thread-block CLUSTER of 8 (co-scheduled blocks, ticket shared through distributed shared memory) pays for
// gang-scheduling eight 43 KB blocks.  Per-block tickets stay.
template <bool WRITE_KEYS>
__global__ void __launch_bounds__(SORT_THREADS)   // (capping at 64 registers for a 4th block per SM measured slower on an earlier GPU)
sort_onesweep_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                     uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, uint32_t n,
                     const uint32_t* __restrict__ n_dev, int shift, uint32_t mask,
                     const uint32_t* __restrict__ hist, uint32_t* status, uint32_t* ticket) {
    __shared__ uint32_t s_wc[SORT_THREADS / 32][RADIX];
    __shared__ uint32_t s_keys[SORT_TILE];
    __shared__ uint32_t s_vals[SORT_TILE];
    __shared__ uint32_t s_gofs[RADIX];
    __shared__ uint32_t s_dstart[RADIX];
    __shared__ uint32_t s_warp[SORT_THREADS / 32];
    __shared__ uint32_t s_bid;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_bid = atomicAdd(ticket, 1u);
#pragma unroll
    for (int i = 0; i < (SORT_THREADS / 32) * RADIX / SORT_THREADS; ++i)
        (&s_wc[0][0])[i * SORT_THREADS + tid] = 0;
    __syncthreads();
    const uint32_t bid = s_bid;
    if (n_dev) n = min(n, *n_dev);                       // count produced on the device; grid sized for the capacity
    if (bid * (uint32_t)SORT_TILE >= n) return;          // nobody looks back at a block past the end
    const uint32_t base = bid * (uint32_t)SORT_TILE + warp * (SORT_ITEMS * 32);

    uint32_t k[SORT_ITEMS];
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        uint32_t idx = base + i * 32 + lane;
        k[i] = idx < n ? keys_in[idx] : 0xFFFFFFFFu;
    }
    // warp-level multisplit ranking; the 16 MATCHes are independent and issued
    // back to back, only the counter updates form a chain
    uint32_t rank[SORT_ITEMS];
    const uint32_t lt = lanemask_lt();
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) rank[i] = __match_any_sync(0xffffffffu, (k[i] >> shift) & mask);
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        const uint32_t d = (k[i] >> shift) & mask;
        const uint32_t peers = rank[i];
        const int leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if (lane == leader) {
            old = s_wc[warp][d];
            s_wc[warp][d] = old + __popc(peers);
        }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[i] = old + __popc(peers & lt);
        __syncwarp();
    }
    // the values are only needed for the scatter; fetching them here (not there) keeps the global round
    // trip off the critical path behind the look-back
    uint32_t v_in[SORT_ITEMS];
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        uint32_t idx = base + i * 32 + lane;
        v_in[i] = idx < n ? vals_in[idx] : 0u;
    }
    __syncthreads();
    // digit tid: exclusive prefix over warps, block count
    uint32_t count = 0;
#pragma unroll
    for (int w = 0; w < SORT_THREADS / 32; ++w) {
        uint32_t c = s_wc[w][tid];
        s_wc[w][tid] = count;
        count += c;
    }
    // publish as early as possible
    uint32_t* my_status = status + (size_t)bid * RADIX + tid;
    st_volatile_u32(my_status, (bid == 0 ? LB_FLAG_INCL : LB_FLAG_AGG) | count);

    const uint32_t dstart = block_excl_scan_256(count, s_warp);
    const uint32_t hexcl = block_excl_scan_256(hist[tid], s_warp);
    s_dstart[tid] = dstart;

    // Decoupled look-back, windowed: LB_WINDOW predecessor words are fetched with
    // independent loads per round trip (one serial L2 hop per predecessor made the
    // chain, not the data movement, the critical path of the pass).
    uint32_t excl = 0;
    if (bid > 0) {
        int p = (int)bid - 1;
        bool done = false;
        while (!done) {
            uint32_t v[LB_WINDOW];
#pragma unroll
            for (int k = 0; k < LB_WINDOW; ++k)
                v[k] = (p - k >= 0) ? ld_volatile_u32(status + (size_t)(p - k) * RADIX + tid) : LB_FLAG_INCL;
#pragma unroll
            for (int k = 0; k < LB_WINDOW; ++k) {
                if (done) break;
                const uint32_t f = v[k] >> 30;
                if (f == 0) {          // not published yet: retry from here
                    p -= k;
                    goto next_round;
                }
                excl += v[k] & LB_VALUE_MASK;
                if (f == 2) done = true;
            }
            p -= LB_WINDOW;
        next_round:;
        }
        st_volatile_u32(my_status, LB_FLAG_INCL | (excl + count));
    }
    s_gofs[tid] = hexcl + excl - dstart;
    __syncthreads();

    // scatter to the block-local digit-sorted order in shared memory
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        uint32_t d = (k[i] >> shift) & mask;
        uint32_t lp = s_dstart[d] + s_wc[warp][d] + rank[i];
        s_keys[lp] = k[i];
        s_vals[lp] = v_in[i];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        uint32_t li = j * SORT_THREADS + tid;
        uint32_t kk = s_keys[li];
        uint32_t d = (kk >> shift) & mask;
        uint32_t pos = s_gofs[d] + li;
        if (pos < n) {
            if (WRITE_KEYS) keys_out[pos] = kk;
            vals_out[pos] = s_vals[li];
        }
    }
}

// Host driver.  Sorts on key bits [begin_bit, end_bit) with ceil(bits/8) passes,
// ping-ponging between (keys_in,vals_in) and (keys_tmp,vals_tmp); the LAST pass
// writes to (keys_final,vals_final) (keys_final may be NULL = don't care).
// `st` must have been carved for >= n items.  Returns the cudaError of the
// launches.
cudaError_t radix_sort_prepare(const SortTemp& st, cudaStream_t stream) {
    return cudaMemsetAsync(st.hist, 0, st.zero_bytes, stream);
}

cudaError_t radix_sort_pairs(uint32_t n, uint32_t* keys_in, uint32_t* vals_in,
                                    uint32_t* keys_tmp, uint32_t* vals_tmp, uint32_t* keys_final,
                                    uint32_t* vals_final, int begin_bit, int end_bit,
                                    const SortTemp& st, cudaStream_t stream, const uint32_t* n_dev,
                                    bool hist_ready, bool prepared, uint32_t* keys_spare) {
    if (n == 0) return cudaSuccess;
    int bits = end_bit - begin_bit;
    int npass = (bits + RADIX_BITS - 1) / RADIX_BITS;
    if (npass < 1) npass = 1;
    if (npass > SORT_MAX_PASSES) return cudaErrorInvalidValue;
    const uint32_t nblk = (uint32_t)div_up64(n, SORT_TILE);
    if (!hist_ready) {
        if (!prepared) {
            cudaError_t e = radix_sort_prepare(st, stream);
            if (e != cudaSuccess) return e;
        }
        if (n_dev) return cudaErrorInvalidValue;       // a device-side count needs a producer-built histogram
        const uint32_t hcap = (uint32_t)device_sm_count() * 8u;
        const uint32_t hgrid = nblk < hcap ? nblk : hcap;
        sort_histogram_kernel<<<hgrid, SORT_THREADS, 0, stream>>>(keys_in, n, begin_bit, end_bit, npass,
                                                                  st.hist);
    }
    uint32_t* src_k = keys_in;
    uint32_t* src_v = vals_in;
    for (int p = 0; p < npass; ++p) {
        const bool last = (p == npass - 1);
        uint32_t* dst_k = last ? keys_final
                          : keys_spare ? (p % 2 == 0 ? keys_tmp : keys_spare)
                                       : (src_k == keys_in ? keys_tmp : keys_in);
        uint32_t* dst_v = last ? vals_final : (src_v == vals_in ? vals_tmp : vals_in);
        int shift = begin_bit + p * RADIX_BITS;
        int pb = end_bit - shift < RADIX_BITS ? end_bit - shift : RADIX_BITS;
        if (pb < 1) pb = 1;
        uint32_t mask = (1u << pb) - 1u;
        uint32_t* status = st.status + (size_t)p * nblk * RADIX;
        if (dst_k)
            sort_onesweep_kernel<true><<<nblk, SORT_THREADS, 0, stream>>>(
                src_k, src_v, dst_k, dst_v, n, n_dev, shift, mask, st.hist + p * RADIX, status, st.tickets + p);
        else
            sort_onesweep_kernel<false><<<nblk, SORT_THREADS, 0, stream>>>(
                src_k, src_v, nullptr, dst_v, n, n_dev, shift, mask, st.hist + p * RADIX, status, st.tickets + p);
        src_k = dst_k;
        src_v = dst_v;
    }
    return cudaGetLastError();
}
#endif  // S3G_RADIX_SORT_IMPL

#ifdef S3G_SCAN_IMPL   // the scan below is compiled by api.cu only
// ---- chained exclusive scan of tiles_touched[order[k]] ---------------------
// Replaces cub::DeviceScan::InclusiveSum (rasterizer_impl.cu:278), but over the
// depth-sorted order and exclusive.  misc[0] = ticket (zeroed), total written to
// *(uint64_t*)(misc + 2).  status: [nblk] zeroed.
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;  // 2048

__global__ void __launch_bounds__(SCAN_THREADS)
scan_tiles_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ tiles_touched,
                  uint32_t n, uint32_t* __restrict__ offsets, uint64_t* status, uint32_t* misc,
                  volatile uint64_t* host_total /*[2] mapped pinned: {total, sequence}*/, uint64_t seq,
                  int use_tickets) {
    __shared__ uint32_t s_warp[SCAN_THREADS / 32];
    __shared__ uint32_t s_bid;
    __shared__ uint64_t s_prefix;
    __shared__ uint64_t s_part[SCAN_THREADS / 32];
    const int tid = threadIdx.x;
    // Block order: a ticket (start order) when the grid is larger than what can be resident at once - a block may
    // only wait on blocks that have started; blockIdx when every block is resident anyway (the host checks): ~1000
    // same-address ticket atomics serialise in L2, which can cost more than the rest of the kernel.
    if (use_tickets) {
        if (tid == 0) s_bid = atomicAdd(&misc[0], 1u);
        __syncthreads();
    }
    const uint32_t bid = use_tickets ? s_bid : blockIdx.x;
    const uint32_t nblk = gridDim.x;
    // blocked arrangement: thread owns SCAN_ITEMS consecutive items
    const uint32_t base = bid * SCAN_TILE + tid * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint32_t sum = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        uint32_t idx = base + i;
        v[i] = idx < n ? tiles_touched[order[idx]] : 0u;
        sum += v[i];
    }
    uint32_t block_total;
    uint32_t texcl = block_excl_scan_256(sum, s_warp, &block_total);
    // Prefix over the preceding blocks.
    uint64_t part = 0;      // 64-bit: the caller rejects counts >= 2^30, but only after it has seen the true total
    if (!use_tickets) {
        // The whole grid is resident (host-checked): publish the block sum, meet at a grid-wide barrier (one arrival
        // counter, ONE polling thread per block), then every thread adds up its share of the preceding sums.  No
        // thread ever polls a neighbour's status word - 250 k threads spinning on L2 lines (the look-back below at
        // one wave) delay the very stores they wait for.
        if (tid == 0) {
            st_volatile_u64(&status[bid], (uint64_t)block_total);
            __threadfence();
            atomicAdd(&misc[1], 1u);
            while (ld_volatile_u32(&misc[1]) < nblk) {}
        }
        __syncthreads();
        for (int idx = tid; idx < (int)bid; idx += SCAN_THREADS) part += ld_volatile_u64(&status[idx]);
    } else {
        // Larger grids: every thread fetches one predecessor's AGGREGATE per window of 256 blocks (independent spin on
        // its own word), the block adds them up: ceil(bid/256) round trips.  Predecessors hold lower tickets, i.e. they
        // have started and publish without waiting on anyone later.
        if (tid == 0) st_volatile_u64(&status[bid], (1ull << 62) | (uint64_t)block_total);
        for (int base = (int)bid - 1; base >= 0; base -= SCAN_THREADS) {
            const int idx = base - tid;
            if (idx >= 0) {
                uint64_t sv;
                do { sv = ld_volatile_u64(&status[idx]); } while ((sv >> 62) == 0);
                part += sv & ((1ull << 62) - 1);
            }
        }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((tid & 31) == 0) s_part[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
        uint64_t excl = 0;
#pragma unroll
        for (int w = 0; w < SCAN_THREADS / 32; ++w) excl += s_part[w];
        s_prefix = excl;
        if (bid == nblk - 1) {
            *reinterpret_cast<uint64_t*>(misc + 2) = excl + block_total;
            if (host_total) {       // the host learns the count without a copy or a stream synchronisation
                host_total[0] = excl + block_total;
                __threadfence_system();
                host_total[1] = seq;
            }
        }
    }
    __syncthreads();
    uint32_t run = (uint32_t)s_prefix + texcl;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        uint32_t idx = base + i;
        if (idx < n) offsets[idx] = run;
        run += v[i];
    }
}

#endif

}  // namespace s3g
