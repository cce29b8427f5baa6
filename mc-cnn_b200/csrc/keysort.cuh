// keysort.cuh -- the block-ordered building blocks of the sparse voxel maps (DESIGN §23, §24), shared by fusion.cu and
// tsdf.cu: block counts and ballot ranks, a 64-bit scan of block counts in block order, a stable LSD radix sort of
// (u64 key, int) pairs, and the binary-search rank of one sorted key array in another.  Every result depends on the element
// order only, never on scheduling, so the maps built from them are the same bit for bit on every run and GPU.
#pragma once

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ITEMS = 8;                         // elements per thread and chunk
constexpr long CHUNK = (long)THREADS * ITEMS;    // elements per block
constexpr int SCAN_THREADS = 1024;
constexpr unsigned FULL = 0xffffffffu;
constexpr int BITS = 8, BINS = 1 << BITS, PASSES = 8;   // 64 bits of key, the top one always 0
static_assert(BINS == THREADS, "one digit per thread in the scatter");

typedef unsigned long long u64;

// the block's sum of k (every thread calls it); valid in thread 0
__device__ __forceinline__ int block_sum(int k, int *warp_n)
{
	k = __reduce_add_sync(FULL, k);
	if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = k;
	__syncthreads();
	int t = 0;
	if (threadIdx.x == 0)
		for (int w = 0; w < THREADS / 32; w++) t += warp_n[w];
	__syncthreads();
	return t;
}

// one round of THREADS elements: this thread's rank among the round's flagged elements before it, and their total
__device__ __forceinline__ int round_rank(bool ok, int *warp_n, int *all)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const unsigned m = __ballot_sync(FULL, ok);
	if (lane == 0) warp_n[warp] = __popc(m);
	__syncthreads();
	int before = __popc(m & ((1u << lane) - 1u)), t = 0;
	for (int w = 0; w < THREADS / 32; w++) {
		const int v = warp_n[w];
		before += w < warp ? v : 0;
		t += v;
	}
	__syncthreads();
	*all = t;
	return before;
}

// off[b] = sum of blk[0 .. b) in 64 bits, *total = the sum of all: each thread scans a contiguous run of blocks
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const int *__restrict__ blk, long long nblk, long long *__restrict__ off,
							    long long *__restrict__ total)
{
	__shared__ long long part[SCAN_THREADS];
	const long long per = (nblk + SCAN_THREADS - 1) / SCAN_THREADS;
	const long long lo = min(nblk, (long long)threadIdx.x * per), hi = min(nblk, lo + per);
	long long s = 0;
	for (long long b = lo; b < hi; b++) s += blk[b];
	part[threadIdx.x] = s;
	__syncthreads();
	if (threadIdx.x == 0) {
		long long a = 0;
		for (int t = 0; t < SCAN_THREADS; t++) {
			const long long v = part[t];
			part[t] = a;
			a += v;
		}
		*total = a;
	}
	__syncthreads();
	s = part[threadIdx.x];
	for (long long b = lo; b < hi; b++) {
		off[b] = s;
		s += blk[b];
	}
}

// ---- stable LSD radix sort of (key, value) ----

// hist[d nblk + b] = the elements of chunk b whose digit is d
__global__ void __launch_bounds__(THREADS) sort_hist_kernel(const u64 *__restrict__ keys, const long long *__restrict__ dn, int shift,
							    int nblk, int *__restrict__ hist)
{
	__shared__ int h[BINS];
	h[threadIdx.x] = 0;
	__syncthreads();
	const long long n = *dn;
	const long base = (long)blockIdx.x * CHUNK;
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		if (e < n) atomicAdd(&h[(int)((keys[e] >> shift) & (BINS - 1))], 1);
	}
	__syncthreads();
	hist[(long)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// each element to hoff[its digit, its block] + the elements of its block and digit before it
__global__ void __launch_bounds__(THREADS) sort_scatter_kernel(const u64 *__restrict__ kin, const int *__restrict__ vin,
							       const long long *__restrict__ dn, int shift, const long long *__restrict__ hoff,
							       int nblk, u64 *__restrict__ kout, int *__restrict__ vout)
{
	__shared__ int wcount[THREADS / 32][BINS];
	__shared__ long long run[BINS];
	const long long n = *dn;
	const long base = (long)blockIdx.x * CHUNK;
	if (base >= n) return;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	run[threadIdx.x] = hoff[(long)threadIdx.x * nblk + blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		__syncthreads();                           // the last round's reads of wcount are done
		for (int b = lane; b < BINS; b += 32) wcount[warp][b] = 0;
		__syncthreads();
		const long e = base + (long)i * THREADS + threadIdx.x;
		const bool ok = e < n;
		u64 k = 0;
		int dg = BINS;                             // no element: a digit of its own
		if (ok) {
			k = kin[e];
			dg = (int)((k >> shift) & (BINS - 1));
		}
		const unsigned peers = __match_any_sync(FULL, dg);
		const int rank = __popc(peers & ((1u << lane) - 1u));
		if (ok && lane == __ffs(peers) - 1) wcount[warp][dg] = __popc(peers);
		__syncthreads();
		if (ok) {
			long long pos = run[dg] + rank;
			for (int w = 0; w < warp; w++) pos += wcount[w][dg];
			kout[pos] = k;
			vout[pos] = vin[e];
		}
		__syncthreads();                           // every read of run before its update
		int t = 0;
		for (int w = 0; w < THREADS / 32; w++) t += wcount[w][threadIdx.x];
		run[threadIdx.x] += t;
	}
}

// the *dn pairs in keyA / valA sorted by key, stably, in PASSES passes that end where they started; keyB / valB, hist
// (BINS nblk ints), hoff (BINS nblk + 1 int64s) and *total (one int64) are scratch, nblk the chunks of the largest *dn
void radix_sort_pairs(u64 *keyA, int *valA, u64 *keyB, int *valB, const long long *dn, int nblk, int *hist, long long *hoff,
		      long long *total, cudaStream_t s)
{
	for (int pass = 0; pass < PASSES; pass++) {
		const bool even = (pass & 1) == 0;
		const u64 *kin = even ? keyA : keyB;
		const int *vin = even ? valA : valB;
		sort_hist_kernel<<<nblk, THREADS, 0, s>>>(kin, dn, BITS * pass, nblk, hist);
		scan_kernel<<<1, SCAN_THREADS, 0, s>>>(hist, (long long)BINS * nblk, hoff, total);
		sort_scatter_kernel<<<nblk, THREADS, 0, s>>>(kin, vin, dn, BITS * pass, hoff, nblk, even ? keyB : keyA, even ? valB : valA);
	}
}

// ---- the rank of sorted keys in a sorted table ----

// the first index in a[0 .. n) whose key is not below k
__device__ __forceinline__ long long lower_bound(const u64 *a, long long n, u64 k)
{
	long long lo = 0, hi = n;
	while (lo < hi) {
		const long long mid = (lo + hi) >> 1;
		if (a[mid] < k)
			lo = mid + 1;
		else
			hi = mid;
	}
	return lo;
}

__device__ __forceinline__ bool fresh(const u64 *tkey, long long n, long long l, u64 k) { return l == n || tkey[l] != k; }

// lb[j] = the rank of frame key j in the table; blk = the chunk's frame keys absent from the table
__global__ void __launch_bounds__(THREADS) match_count_kernel(const u64 *__restrict__ fkey, const long long *__restrict__ dU,
							      const u64 *__restrict__ tkey, long long n, long long *__restrict__ lb,
							      int *__restrict__ blk)
{
	__shared__ int warp_n[THREADS / 32];
	const long long U = *dU;
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0;
	for (int i = 0; i < ITEMS; i++) {
		const long j = base + (long)i * THREADS + threadIdx.x;
		if (j < U) {
			const long long l = lower_bound(tkey, n, fkey[j]);
			lb[j] = l;
			k += fresh(tkey, n, l, fkey[j]);
		}
	}
	k = block_sum(k, warp_n);
	if (threadIdx.x == 0) blk[blockIdx.x] = k;
}

// nn[j] = the frame keys before j that are absent from the table
__global__ void __launch_bounds__(THREADS) match_rank_kernel(const u64 *__restrict__ fkey, const long long *__restrict__ dU,
							     const u64 *__restrict__ tkey, long long n, const long long *__restrict__ lb,
							     const long long *__restrict__ off, long long *__restrict__ nn)
{
	__shared__ int warp_n[THREADS / 32];
	const long long U = *dU;
	const long base = (long)blockIdx.x * CHUNK;
	long long at = off[blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		const long j = base + (long)i * THREADS + threadIdx.x;
		const bool ok = j < U && fresh(tkey, n, lb[j], fkey[j]);
		int all;
		const int r = round_rank(ok, warp_n, &all);
		if (j < U) nn[j] = at + r;
		at += all;
	}
}

long grid_for(long long n) { return std::max<long>(1, std::min<long long>((n + THREADS - 1) / THREADS, (long long)adc_num_sms() * 8)); }

}  // namespace
