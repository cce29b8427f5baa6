// mb_eval.cu -- the MiddEval3 SDK's evaldisp metrics and the A50-A99 error quantiles of one map, for sm_90a
// (mccnn_mb_evaldisp).
//
// Per ground-truth pixel (x, y) with gt != +inf: d = (float)scale * disp[y / scale][x / scale]; valid when d != +inf; a valid
// d is clamped as max(0, min(maxd, d)) with the SDK's ternary macros (NaN stays NaN, -inf becomes 0); err = |d - gt| in fp32.
// Region 0 (nonocc) takes the pixels whose mask byte is 255 (every pixel without a mask), region 1 (all) every pixel.
//
// Launches on the stream, nothing read back and nothing allocated:
// * score: each block takes the chunks blockIdx.x, + gridDim.x, ... of 4096 pixels, the grid fixed by the pixel count
//   alone.  Integer counts by warp sums and integer atomics; sum(err) and sum(err^2) in float64, in a fixed order per thread,
//   then a fixed tree per block, to a per-block slot (no float atomics, so the same bits on every run and every GPU).  The
//   same pass builds the 256-bin histogram of the top byte of every valid err, per region: radix select's first pass;
// * finish: one block adds the block sums in a fixed order;
// * quantiles: exact radix select on the err's bit pattern (non-negative floats and fabsf's positive NaN order like their
//   uint32 bits).  For each of the 8 (region, q) targets a one-block pick kernel finds the bin that holds the target's rank,
//   appends it to the target's prefix and narrows the rank; then a histogram pass over the pixels (err recomputed, no
//   n-sized buffer) counts the next byte of the keys that match each prefix.  Targets of one region with equal prefixes
//   share one histogram.  Four 8-bit digits: pick, (hist, pick) x 3.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ITEMS = 16;                        // pixels per thread and chunk
constexpr long CHUNK = (long)THREADS * ITEMS;    // pixels per chunk
constexpr int MAX_BLOCKS = 1024;                 // the grid of the pixel passes (block sums kept in the scratch)
constexpr int NQ = 4;                            // A50, A90, A95, A99
constexpr int NT = 2 * NQ;                       // (region, q) targets
constexpr unsigned FULL = 0xffffffffu;
__constant__ int PERCENT[NQ] = {50, 90, 95, 99};

// the caller's scratch: block sums, then the select state
struct Scratch {
	double part[MAX_BLOCKS][4];              // per block: sum(err), sum(err^2) of region 0, then of region 1
	unsigned hist[NT][256];                  // target t's histogram of the current digit (shared: see src)
	unsigned prefix[NT];                     // the key bits found so far
	unsigned rank[NT];                       // the target's 1-based rank among the keys that match the prefix
	int src[NT];                             // the target whose histogram serves t in this digit, -1 = no valid pixel
};
static_assert(sizeof(Scratch) <= MCCNN_MB_EVAL_SCRATCH_BYTES, "MCCNN_MB_EVAL_SCRATCH_BYTES is too small");

struct Geometry {
	const float *disp;
	const float *gt;
	const unsigned char *mask;
	int w, Wg, scale;
	long n;                                  // Hg * Wg
	float maxd;
};

// one ground-truth pixel: whether it counts (gt != inf), its regions, validity and err
struct Pixel {
	bool known, nonocc, valid;
	float err;
};

__device__ __forceinline__ Pixel pixel(const Geometry &g, long p)
{
	Pixel px;
	const float t = g.gt[p];
	px.known = t != CUDART_INF_F;
	const int y = (int)(p / g.Wg), x = (int)(p - (long)y * g.Wg);
	float d = __fmul_rn((float)g.scale, g.disp[(long)(y / g.scale) * g.w + x / g.scale]);
	px.valid = d != CUDART_INF_F;
	if (px.valid) {
		d = (g.maxd < d) ? g.maxd : d;   // min(maxd, d)
		d = (0.f > d) ? 0.f : d;         // max(0, d)
	}
	px.err = fabsf(__fsub_rn(d, t));
	px.nonocc = px.known && (!g.mask || g.mask[p] == 255);
	return px;
}

// add 1 to bin `bin` of the shared histogram h for the lanes with `in`, one atomic per distinct bin in the warp
__device__ __forceinline__ void warp_hist_add(unsigned *h, bool in, unsigned bin)
{
	const unsigned peers = __match_any_sync(FULL, in ? bin : 0xffffffffu);
	if (in && (__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(h + bin, __popc(peers));
}

__device__ __forceinline__ long chunk_base(int c) { return (long)c * CHUNK; }

// counts, block sums and the first digit's histograms (slot 0 region 0, slot NQ region 1)
__global__ void __launch_bounds__(THREADS) score_kernel(Geometry g, int nchunk, unsigned long long *__restrict__ counts,
							 Scratch *__restrict__ sc)
{
	__shared__ unsigned block_counts[2 * MCCNN_MB_NCOUNT];
	__shared__ unsigned hist[2][256];
	__shared__ double sh[4][THREADS];
	const int tid = threadIdx.x;
	if (tid < 2 * MCCNN_MB_NCOUNT) block_counts[tid] = 0;
	hist[0][tid] = hist[1][tid] = 0;
	__syncthreads();

	unsigned c[2][MCCNN_MB_NCOUNT];
	double s[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
	for (int r = 0; r < 2; r++)
#pragma unroll
		for (int k = 0; k < MCCNN_MB_NCOUNT; k++) c[r][k] = 0;

	for (int ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
		for (int i = 0; i < ITEMS; i++) {             // uniform trip count: warp_hist_add needs every lane
			const long p = chunk_base(ch) + (long)i * THREADS + tid;
			Pixel px = {false, false, false, 0.f};
			if (p < g.n) px = pixel(g, p);
			const unsigned key = __float_as_uint(px.err), bin = key >> 24;
#pragma unroll
			for (int r = 0; r < 2; r++) {
				const bool in = r ? px.known : px.nonocc;
				warp_hist_add(hist[r], in && px.valid, bin);
				if (!in) continue;
				c[r][MCCNN_MB_N]++;
				if (!px.valid) {
					c[r][MCCNN_MB_INVALID]++;
					continue;
				}
				const float e = px.err;
				c[r][MCCNN_MB_VALID]++;
				c[r][MCCNN_MB_BAD05] += e > 0.5f;
				c[r][MCCNN_MB_BAD1] += e > 1.f;
				c[r][MCCNN_MB_BAD2] += e > 2.f;
				c[r][MCCNN_MB_BAD4] += e > 4.f;
				const double ed = (double)e;
				s[r][0] = __dadd_rn(s[r][0], ed);
				s[r][1] = __dadd_rn(s[r][1], __dmul_rn(ed, ed));   // exact: a float's square fits a double
			}
		}
	}
#pragma unroll
	for (int r = 0; r < 2; r++)
#pragma unroll
		for (int k = 0; k < MCCNN_MB_NCOUNT; k++) {
			const unsigned wsum = __reduce_add_sync(FULL, c[r][k]);
			if ((tid & 31) == 0 && wsum) atomicAdd(&block_counts[r * MCCNN_MB_NCOUNT + k], wsum);
		}
#pragma unroll
	for (int k = 0; k < 4; k++) sh[k][tid] = s[k >> 1][k & 1];
	__syncthreads();
	if (tid < 2 * MCCNN_MB_NCOUNT && block_counts[tid]) atomicAdd(counts + tid, (unsigned long long)block_counts[tid]);
	for (int r = 0; r < 2; r++)
		if (hist[r][tid]) atomicAdd(&sc->hist[r * NQ][tid], hist[r][tid]);
	for (int h = THREADS / 2; h; h >>= 1) {       // a fixed tree
		if (tid < h)
#pragma unroll
			for (int k = 0; k < 4; k++) sh[k][tid] = __dadd_rn(sh[k][tid], sh[k][tid + h]);
		__syncthreads();
	}
	if (tid < 4) sc->part[blockIdx.x][tid] = sh[tid][0];
}

// sums[r][k] = the block sums added in a fixed order: thread t over blocks t, t + THREADS, ..., then a tree
__global__ void __launch_bounds__(THREADS) finish_kernel(const Scratch *__restrict__ sc, int nblk, double *__restrict__ sums)
{
	__shared__ double sh[4][THREADS];
	const int tid = threadIdx.x;
	double a[4] = {0.0, 0.0, 0.0, 0.0};
	for (int b = tid; b < nblk; b += THREADS)
#pragma unroll
		for (int k = 0; k < 4; k++) a[k] = __dadd_rn(a[k], sc->part[b][k]);
#pragma unroll
	for (int k = 0; k < 4; k++) sh[k][tid] = a[k];
	__syncthreads();
	for (int h = THREADS / 2; h; h >>= 1) {
		if (tid < h)
#pragma unroll
			for (int k = 0; k < 4; k++) sh[k][tid] = __dadd_rn(sh[k][tid], sh[k][tid + h]);
		__syncthreads();
	}
	if (tid < 4) sums[tid] = sh[tid][0];
}

// One digit of the select, one warp per target: the bin of hist[src[t]] that holds rank[t] extends prefix[t]; then the
// histograms are cleared and src set up for the next digit.  Digit 0 starts the targets from the counts; digit 3 writes the
// quantiles.  Within the launch a target's state lives in registers, the same in every lane of its warp; `sc` is read after
// a barrier for what other warps wrote, so it is not __restrict__ (that let the compiler hoist such loads above it).
__global__ void __launch_bounds__(NT * 32) pick_kernel(Scratch *sc, const unsigned long long *__restrict__ counts, int digit,
						      float *__restrict__ quantiles)
{
	const int t = threadIdx.x >> 5, lane = threadIdx.x & 31, r = t / NQ;
	const int shift = 24 - 8 * digit;
	int src;
	unsigned prefix, rank;
	if (digit == 0) {
		const unsigned long long nvalid = counts[r * MCCNN_MB_NCOUNT + MCCNN_MB_VALID];
		src = nvalid ? r * NQ : -1;
		prefix = 0;
		rank = (unsigned)((PERCENT[t % NQ] * nvalid + 99) / 100);           // ceil(q nvalid), exact
	} else {
		src = sc->src[t];
		prefix = sc->prefix[t];
		rank = sc->rank[t];
	}
	if (src >= 0) {
		unsigned v[8], sum = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) sum += v[j] = sc->hist[src][lane * 8 + j];
		unsigned incl = sum;                        // inclusive scan over the lanes
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const unsigned y = __shfl_up_sync(FULL, incl, o);
			if (lane >= o) incl += y;
		}
		const unsigned excl = incl - sum;
		const unsigned owner = __ballot_sync(FULL, excl < rank && rank <= incl);
		const int o = owner ? __ffs(owner) - 1 : 0;    // the lane whose bins hold the rank (always one)
		if (lane == o) {
			unsigned before = excl;
			int bin = 7;
#pragma unroll
			for (int j = 0; j < 7; j++) {
				if (bin == 7 && before + v[j] >= rank) bin = j;
				if (bin == 7) before += v[j];
			}
			prefix |= (unsigned)(lane * 8 + bin) << shift;
			rank -= before;
		}
		prefix = __shfl_sync(FULL, prefix, o);
		rank = __shfl_sync(FULL, rank, o);
	}
	if (lane == 0) {
		sc->prefix[t] = prefix;
		sc->rank[t] = rank;
	}
	__syncthreads();                                    // every warp has read its histogram and stored its prefix
	for (int i = threadIdx.x; i < NT * 256; i += blockDim.x) (&sc->hist[0][0])[i] = 0;
	if (digit == 3) {
		if (lane == 0) quantiles[t] = src >= 0 ? __uint_as_float(prefix) : CUDART_NAN_F;
		return;
	}
	if (lane == 0) {                                    // the first target of the region with the same prefix
		int s = src;
		if (src >= 0)
			for (s = r * NQ; s < t; s++)
				if (sc->prefix[s] == prefix) break;
		sc->src[t] = s;
	}
}

// digit `digit` (1..3) of the keys that match each target's prefix in its top 8 * digit bits
__global__ void __launch_bounds__(THREADS) hist_kernel(Geometry g, int nchunk, Scratch *__restrict__ sc, int digit)
{
	__shared__ unsigned hist[NT][256];
	__shared__ unsigned prefix[NT];
	__shared__ int src[NT];
	const int tid = threadIdx.x;
	for (int i = tid; i < NT * 256; i += THREADS) (&hist[0][0])[i] = 0;
	if (tid < NT) {
		prefix[tid] = sc->prefix[tid];
		src[tid] = sc->src[tid];
	}
	__syncthreads();
	const int hi = 32 - 8 * digit, shift = hi - 8;
	for (int ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
		for (int i = 0; i < ITEMS; i++) {
			const long p = chunk_base(ch) + (long)i * THREADS + tid;
			Pixel px = {false, false, false, 0.f};
			if (p < g.n) px = pixel(g, p);
			const unsigned key = __float_as_uint(px.err), bin = (key >> shift) & 255u;
#pragma unroll
			for (int t = 0; t < NT; t++) {
				if (src[t] != t) continue;          // the same for every lane
				const bool in = (t < NQ ? px.nonocc : px.known) && px.valid && (key >> hi) == (prefix[t] >> hi);
				warp_hist_add(hist[t], in, bin);
			}
		}
	}
	__syncthreads();
	for (int t = 0; t < NT; t++)
		if (src[t] == t && hist[t][tid]) atomicAdd(&sc->hist[t][tid], hist[t][tid]);
}

}  // namespace

extern "C" int mccnn_mb_evaldisp(const float *disp, int h, int w, const float *gt, int Hg, int Wg, const unsigned char *mask,
				 int maxdisp, long long *counts, double *sums, float *quantiles, void *scratch,
				 adcensus_stream_t stream)
{
	if (!disp || !gt || !counts || !sums || !quantiles || !scratch || h < 1 || w < 1 || maxdisp < 1) return ADCENSUS_EINVAL;
	const int scale = Wg / w;
	if ((scale != 1 && scale != 2 && scale != 4) || Wg != scale * w || (long)Hg != (long)scale * h) return ADCENSUS_EINVAL;
	const long n = (long)Hg * Wg;
	if (n >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	Scratch *sc = (Scratch *)scratch;
	const Geometry g = {disp, gt, mask, w, Wg, scale, n, (float)((long)scale * maxdisp)};
	const int nchunk = adc_div_up(n, CHUNK), nblk = std::min(nchunk, MAX_BLOCKS);
	ADC_CUDA(cudaMemsetAsync(counts, 0, sizeof(long long) * 2 * MCCNN_MB_NCOUNT, s));
	ADC_CUDA(cudaMemsetAsync(sc->hist, 0, sizeof(sc->hist), s));
	score_kernel<<<nblk, THREADS, 0, s>>>(g, nchunk, (unsigned long long *)counts, sc);
	ADC_CHECK_LAUNCH();
	finish_kernel<<<1, THREADS, 0, s>>>(sc, nblk, sums);
	ADC_CHECK_LAUNCH();
	for (int digit = 0; digit < 4; digit++) {
		if (digit) {
			hist_kernel<<<nblk, THREADS, 0, s>>>(g, nchunk, sc, digit);
			ADC_CHECK_LAUNCH();
		}
		pick_kernel<<<1, NT * 32, 0, s>>>(sc, (const unsigned long long *)counts, digit, quantiles);
		ADC_CHECK_LAUNCH();
	}
	return 0;
}
