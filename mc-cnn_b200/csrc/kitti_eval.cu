// kitti_eval.cu -- the KITTI 2012 / 2015 devkits' stereo metrics for one estimate, for sm_90a (mccnn_kitti_devkit_counts).
//
// Four steps on the stream, all per pixel or per row, nothing read back:
// * quantise: the float map as dataio.write_png16 stores it (or the stored uint16 values) -> the devkit's estimate, -1 where
//   invalid, plus a byte of the original validity (density needs it after the interpolation has filled the holes);
// * rows: one warp per row, two sweeps over 32-pixel chunks.  Left to right every invalid pixel takes the value of the
//   nearest valid pixel to its left (or stays -1); right to left it takes min(that, the nearest valid value to its right),
//   or the right one alone where there is no left one.  That is the devkit's sequence of interior fill, left and right
//   extrapolation in closed form: a run with valid pixels on both sides gets the min of the two, a run touching one end of
//   the row the value of the valid pixel on its other side.  A row with a valid pixel ends fully valid, so the first and
//   last such rows are the only ones the column pass reads (integer atomics);
// * columns: the rows above the first valid row copy it, those below the last valid row copy it; fully invalid rows in
//   between stay -1, as in the devkit;
// * score: per pixel with ground truth the integer counts of include/adcensus_b200.h (warp sums, then integer atomics)
//   and e in float64.  Every block sums a fixed range of 4096 pixels in a fixed order, one block then adds the block sums in
//   a fixed order: no float atomics, and the same bits on every run and every GPU whatever its SM count.
#include <climits>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ITEMS = 16;                        // pixels per thread in the score kernel
constexpr long CHUNK = (long)THREADS * ITEMS;    // pixels per score block
constexpr unsigned FULL = 0xffffffffu;

// dataio.write_png16's value of one float: d < 1e-5 -> 0, else the fp32 product d * 256 truncated and clamped to 65535;
// NaN -> 0 (what numpy's conversion gives on x86)
__device__ __forceinline__ unsigned png16_value(float d)
{
	if (!(d >= 1e-5f)) return 0;
	const float p = __fmul_rn(d, 256.f);
	return p >= 65535.f ? 65535u : __float2uint_rz(p);
}

// the devkit's estimate (-1 = invalid) and validity of every pixel; block 0 also resets the first / last valid row
__global__ void quantise_kernel(const float *__restrict__ disp, const unsigned short *__restrict__ disp16, long n,
				float *__restrict__ est, unsigned char *__restrict__ valid, int *__restrict__ rows)
{
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		rows[0] = INT_MAX;
		rows[1] = -1;
	}
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		const unsigned v = disp ? png16_value(disp[p]) : (unsigned)disp16[p];
		est[p] = v ? __fmul_rn((float)v, 1.f / 256.f) : -1.f;     // exact
		valid[p] = v != 0;
	}
}

// interpolateBackground's row steps on one row per warp, in place
__global__ void row_kernel(float *__restrict__ ipol, const unsigned char *__restrict__ valid, int H, int W, int *__restrict__ rows)
{
	const int lane = threadIdx.x & 31;
	const int v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (v >= H) return;                           // the whole warp
	float *row = ipol + (long)v * W;
	const unsigned char *ok = valid + (long)v * W;

	// left to right: an invalid pixel takes the nearest valid value on its left, -1 if there is none
	float carry = -1.f;
	for (int u0 = 0; u0 < W; u0 += 32) {
		const int u = u0 + lane;
		const bool in = u < W, val = in && ok[u];
		const float x = in ? row[u] : -1.f;
		const unsigned m = __ballot_sync(FULL, val);
		const unsigned below = m & ((1u << lane) - 1u);
		const float y = __shfl_sync(FULL, x, below ? 31 - __clz(below) : lane);
		if (in && !val) row[u] = below ? y : carry;
		if (m) carry = __shfl_sync(FULL, x, 31 - __clz(m));
	}
	if (carry < 0.f) return;                      // no valid pixel: the row stays -1 (carry is the same in every lane)
	if (lane == 0) {
		atomicMin(rows, v);
		atomicMax(rows + 1, v);
	}

	// right to left: with a valid pixel on the right, the min of both sides, or the right one where the left is -1
	carry = -1.f;
	for (int u0 = (W - 1) / 32 * 32; u0 >= 0; u0 -= 32) {
		const int u = u0 + lane;
		const bool in = u < W, val = in && ok[u];
		const float x = in ? row[u] : -1.f;
		const unsigned m = __ballot_sync(FULL, val);
		const unsigned above = lane == 31 ? 0u : m & (FULL << (lane + 1));
		const float y = __shfl_sync(FULL, x, above ? __ffs(above) - 1 : lane);
		const float r = above ? y : carry;
		if (in && !val && r >= 0.f) row[u] = x >= 0.f ? fminf(x, r) : r;
		if (m) carry = __shfl_sync(FULL, x, __ffs(m) - 1);
	}
}

// interpolateBackground's column steps: rows above the first valid row copy it, rows below the last one copy that
__global__ void column_kernel(float *__restrict__ ipol, const int *__restrict__ rows, int W, long n)
{
	const int first = rows[0], last = rows[1];
	if (last < 0) return;                         // no valid pixel at all
	const long lo = (long)first * W, hi = (long)(last + 1) * W;
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		if (p < lo) ipol[p] = ipol[lo + p % W];
		else if (p >= hi) ipol[p] = ipol[(long)last * W + p % W];
	}
}

// the counts of the pixels [blockIdx.x * CHUNK, + CHUNK), added to counts; the block's two e sums to part[2 blockIdx.x + r]
__global__ void __launch_bounds__(THREADS) score_kernel(const float *__restrict__ ipol, const unsigned char *__restrict__ valid,
							 const unsigned short *__restrict__ gt_noc,
							 const unsigned short *__restrict__ gt_occ,
							 const unsigned char *__restrict__ obj, long n,
							 unsigned long long *__restrict__ counts, double *__restrict__ part)
{
	__shared__ unsigned block_counts[2 * MCCNN_KITTI_NCOUNT];
	__shared__ double sh[2][THREADS];
	const int tid = threadIdx.x;
	if (tid < 2 * MCCNN_KITTI_NCOUNT) block_counts[tid] = 0;

	unsigned c[2][MCCNN_KITTI_NCOUNT];
	double s[2] = {0.0, 0.0};
#pragma unroll
	for (int r = 0; r < 2; r++)
#pragma unroll
		for (int k = 0; k < MCCNN_KITTI_NCOUNT; k++) c[r][k] = 0;

	const long base = (long)blockIdx.x * CHUNK;
#pragma unroll 4
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + tid;
		if (p >= n) break;
		const float d = ipol[p];
		const unsigned dense = valid[p];
		const bool fg = obj && obj[p];
#pragma unroll
		for (int r = 0; r < 2; r++) {
			const unsigned g = (r ? gt_occ : gt_noc)[p];
			if (!g) continue;
			const float dg = __fmul_rn((float)g, 1.f / 256.f);         // exact
			const float e = fabsf(__fsub_rn(dg, d));
			const bool d1 = e > 3.f && __fdiv_rn(e, dg) > 0.05f;
			c[r][MCCNN_KITTI_GT]++;
			c[r][MCCNN_KITTI_DENSE] += dense;
			c[r][MCCNN_KITTI_OUT2] += e > 2.f;
			c[r][MCCNN_KITTI_OUT3] += e > 3.f;
			c[r][MCCNN_KITTI_OUT4] += e > 4.f;
			c[r][MCCNN_KITTI_OUT5] += e > 5.f;
			c[r][fg ? MCCNN_KITTI_D1_FG : MCCNN_KITTI_D1_BG] += d1;
			c[r][fg ? MCCNN_KITTI_GT_FG : MCCNN_KITTI_GT_BG]++;
			s[r] = __dadd_rn(s[r], (double)e);
		}
	}
	__syncthreads();                              // block_counts zeroed
#pragma unroll
	for (int r = 0; r < 2; r++)
#pragma unroll
		for (int k = 0; k < MCCNN_KITTI_NCOUNT; k++) {
			const unsigned w = __reduce_add_sync(FULL, c[r][k]);
			if ((tid & 31) == 0 && w) atomicAdd(&block_counts[r * MCCNN_KITTI_NCOUNT + k], w);
		}
	sh[0][tid] = s[0];
	sh[1][tid] = s[1];
	__syncthreads();
	if (tid < 2 * MCCNN_KITTI_NCOUNT && block_counts[tid])
		atomicAdd(counts + tid, (unsigned long long)block_counts[tid]);
	for (int h = THREADS / 2; h; h >>= 1) {       // a fixed tree
		if (tid < h) {
			sh[0][tid] = __dadd_rn(sh[0][tid], sh[0][tid + h]);
			sh[1][tid] = __dadd_rn(sh[1][tid], sh[1][tid + h]);
		}
		__syncthreads();
	}
	if (tid < 2) part[2 * blockIdx.x + tid] = sh[tid][0];
}

// sums[r] = the block sums of region r added in a fixed order: thread t over blocks t, t + THREADS, ..., then a tree
__global__ void __launch_bounds__(THREADS) finish_kernel(const double *__restrict__ part, int nblk, double *__restrict__ sums)
{
	__shared__ double sh[2][THREADS];
	const int tid = threadIdx.x;
	double a = 0.0, b = 0.0;
	for (int k = tid; k < nblk; k += THREADS) {
		a = __dadd_rn(a, part[2 * k]);
		b = __dadd_rn(b, part[2 * k + 1]);
	}
	sh[0][tid] = a;
	sh[1][tid] = b;
	__syncthreads();
	for (int h = THREADS / 2; h; h >>= 1) {
		if (tid < h) {
			sh[0][tid] = __dadd_rn(sh[0][tid], sh[0][tid + h]);
			sh[1][tid] = __dadd_rn(sh[1][tid], sh[1][tid + h]);
		}
		__syncthreads();
	}
	if (tid < 2) sums[tid] = sh[tid][0];
}

long grid_for(long n) { return std::min<long>((n + THREADS - 1) / THREADS, (long)adc_num_sms() * 8); }

int devkit_counts(const float *disp, const unsigned short *disp16, const unsigned short *gt_noc, const unsigned short *gt_occ,
		  const unsigned char *obj, int H, int W, float *ipol, long long *counts, double *sums, char *scratch,
		  cudaStream_t s)
{
	const long n = (long)H * W;
	const int nblk = adc_div_up(n, CHUNK);
	double *part = (double *)scratch;
	int *rows = (int *)(scratch + sizeof(double) * 2 * nblk);
	float *est = ipol ? ipol : (float *)(rows + 4);
	unsigned char *valid = (unsigned char *)(rows + 4) + (ipol ? 0 : sizeof(float) * n);
	ADC_CUDA(cudaMemsetAsync(counts, 0, sizeof(long long) * 2 * MCCNN_KITTI_NCOUNT, s));
	quantise_kernel<<<grid_for(n), THREADS, 0, s>>>(disp, disp16, n, est, valid, rows);
	ADC_CHECK_LAUNCH();
	row_kernel<<<adc_div_up(H, THREADS / 32), THREADS, 0, s>>>(est, valid, H, W, rows);
	ADC_CHECK_LAUNCH();
	column_kernel<<<grid_for(n), THREADS, 0, s>>>(est, rows, W, n);
	ADC_CHECK_LAUNCH();
	score_kernel<<<nblk, THREADS, 0, s>>>(est, valid, gt_noc, gt_occ, obj, n, (unsigned long long *)counts, part);
	ADC_CHECK_LAUNCH();
	finish_kernel<<<1, THREADS, 0, s>>>(part, nblk, sums);
	ADC_CHECK_LAUNCH();
	return 0;
}

}  // namespace

extern "C" int mccnn_kitti_devkit_counts(const float *disp, const unsigned short *disp16, const unsigned short *gt_noc,
					 const unsigned short *gt_occ, const unsigned char *obj_map, int H, int W, float *ipol,
					 long long *counts, double *sums, adcensus_stream_t stream)
{
	if (!disp == !disp16 || !gt_noc || !gt_occ || !counts || !sums || H < 1 || W < 1) return ADCENSUS_EINVAL;
	const long n = (long)H * W;
	if (n >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	// block sums, the first / last valid row (4 ints keep what follows 16-byte aligned), the estimate unless the caller
	// keeps it in ipol, the validity bytes
	const size_t bytes = sizeof(double) * 2 * adc_div_up(n, CHUNK) + sizeof(int) * 4 + (ipol ? 0 : sizeof(float) * n) + n;
	char *scratch = nullptr;
	int rc = adc_scratch_alloc((void **)&scratch, bytes, s);
	if (rc) return rc;
	rc = devkit_counts(disp, disp16, gt_noc, gt_occ, obj_map, H, W, ipol, counts, sums, scratch, s);
	const int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}
