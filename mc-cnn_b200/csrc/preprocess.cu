// preprocess.cu -- label cleaning of KITTI disparity maps and the training-sample lists of preprocess_kitti.lua, for sm_90a.
//
// Reference: remove_nonvisible adcensus.cu:1723-1745, remove_occluded :1747-1771, remove_white :1773-1796, make_dataset2
// :1900-1929 (a host loop there), driven by preprocess_kitti.lua:95-116.
//
// remove_occluded is a row scan instead of the reference's O(W) loop per pixel.  With a_j = j - y_j, pixel x is occluded iff
// min over j > x of a_j < a_x (strict).  The reference's threads read neighbours that others may be zeroing at the same time;
// zeroing raises a_j (y >= 0), and the pixel attaining the suffix minimum is never zeroed itself, so the reference's result
// is the same as deciding every pixel on the values before the call -- which one reverse suffix minimum per row computes.
// Both comparisons are exact (hence identical) when every x - y is exact in fp32: maps read by readPNG16 (multiples of 1/256
// in [0, 256)) with W <= 2^15.  DESIGN.md has the argument in full.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int PP_THREADS = 256;          // one block per row; thread t owns the contiguous chunk [t * per, (t + 1) * per)
constexpr int PP_WARPS = PP_THREADS / 32;
constexpr int SCAN_THREADS = 1024;
constexpr int MAX_W = 1 << 15;           // exactness bound of the suffix-min rule, and the row fits in shared memory

enum { ROW_OCCLUDED = 0, ROW_COUNT = 1, ROW_FILL = 2 };

__global__ void nonvisible_kernel(float *__restrict__ y, size_t n, int W)
{
	for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < n; id += (size_t)gridDim.x * blockDim.x) {
		int x = (int)(id % W);
		if (y[id] >= x) y[id] = 0;                                      // :1728
	}
}

__global__ void white_kernel(const float *__restrict__ x, float *__restrict__ y, size_t n)
{
	for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < n; id += (size_t)gridDim.x * blockDim.x)
		if (x[id] == 255) y[id] = 0;                                    // :1778
}

// min over the chunks of the threads AFTER this one (+inf for the last thread)
__device__ float block_suffix_min_exclusive(float v, float *sh)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	float inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		float t = __shfl_down_sync(0xffffffffu, inc, o);
		if (lane + o < 32) inc = fminf(inc, t);
	}
	if (lane == 0) sh[warp] = inc;
	float exc = __shfl_down_sync(0xffffffffu, inc, 1);
	if (lane == 31) exc = CUDART_INF_F;
	__syncthreads();
	for (int w = warp + 1; w < PP_WARPS; w++) exc = fminf(exc, sh[w]);
	__syncthreads();
	return exc;
}

// sum over the threads BEFORE this one; *total receives the block's sum
__device__ int block_prefix_sum_exclusive(int v, int *sh, int *total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	int inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		int t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= o) inc += t;
	}
	if (lane == 31) sh[warp] = inc;
	__syncthreads();
	int base = 0, all = 0;
	for (int w = 0; w < PP_WARPS; w++) {
		if (w < warp) base += sh[w];
		all += sh[w];
	}
	__syncthreads();
	*total = all;
	return base + inc - v;
}

// One block per map row r = i * H + row.  ROW_OCCLUDED: y <- remove_occluded(y) in place.  ROW_COUNT / ROW_FILL: a copy of
// disp's row in shared memory goes through remove_nonvisible, remove_occluded and remove_white (against x0); then the number
// of entries > 0.5 goes to count[r] (ROW_COUNT), or the entries are written as (i + 1, row, x, d) float rows at the row's
// offset in nnz_tr / nnz_te (ROW_FILL), in ascending x -- make_dataset2's order.
template <int MODE>
__global__ void __launch_bounds__(PP_THREADS) rows_kernel(float *__restrict__ y, const float *__restrict__ disp,
							  const float *__restrict__ x0, const int *__restrict__ is_te, int H,
							  int W, int *__restrict__ count, const int *__restrict__ off_tr,
							  const int *__restrict__ off_te, float *__restrict__ nnz_tr,
							  long long cap_tr, float *__restrict__ nnz_te, long long cap_te)
{
	extern __shared__ float row[];
	__shared__ float shf[PP_WARPS];
	__shared__ int shi[PP_WARPS];
	const size_t r = blockIdx.x;
	const size_t base = r * (size_t)W;
	const int per = (W + PP_THREADS - 1) / PP_THREADS;
	const int xa = min(W, (int)threadIdx.x * per), xb = min(W, xa + per);

	for (int x = threadIdx.x; x < W; x += PP_THREADS) {
		float v = MODE == ROW_OCCLUDED ? y[base + x] : disp[base + x];
		if (MODE != ROW_OCCLUDED && v >= x) v = 0;                      // remove_nonvisible
		row[x] = v;
	}
	__syncthreads();

	// remove_occluded: exclusive suffix minimum of a_j = j - y_j, chunk by chunk, then inside the chunk backwards
	float m = CUDART_INF_F;
	for (int x = xa; x < xb; x++) m = fminf(m, (float)x - row[x]);
	float suf = block_suffix_min_exclusive(m, shf);
	for (int x = xb - 1; x >= xa; x--) {
		float a = (float)x - row[x];
		if (suf < a) row[x] = 0;
		suf = fminf(suf, a);
	}
	__syncthreads();

	if constexpr (MODE == ROW_OCCLUDED) {
		for (int x = threadIdx.x; x < W; x += PP_THREADS) y[base + x] = row[x];
	} else {
		for (int x = threadIdx.x; x < W; x += PP_THREADS)                     // remove_white, after the occlusion decisions
			if (x0[base + x] == 255) row[x] = 0;
		__syncthreads();

		int c = 0;
		for (int x = xa; x < xb; x++) c += row[x] > 0.5f;                     // make_dataset2's test, adcensus.cu:1917
		int total = 0;
		int before = block_prefix_sum_exclusive(c, shi, &total);
		if constexpr (MODE == ROW_COUNT) {
			if (threadIdx.x == 0) count[r] = total;
		} else {
			const int i = (int)(r / H);
			const bool te = is_te[i] != 0;
			float *out = te ? nnz_te : nnz_tr;
			const long long cap = te ? cap_te : cap_tr;
			long long t = (long long)(te ? off_te : off_tr)[r] + before;
			const float img = (float)(i + 1), yy = (float)(int)(r % H);
			for (int x = xa; x < xb; x++) {
				float d = row[x];
				if (d > 0.5f) {
					if (t < cap) *reinterpret_cast<float4 *>(out + 4 * t) = make_float4(img, yy, (float)x, d);
					t++;
				}
			}
		}
	}
}

// Exclusive scans of the per-row counts, separately over the rows of training images (is_te 0) and validation images
// (is_te 1), in row order; totals[0] / totals[1] receive the two sums.  One block.
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const int *__restrict__ count, const int *__restrict__ is_te,
							    int R, int H, int *__restrict__ off_tr, int *__restrict__ off_te,
							    long long *__restrict__ totals)
{
	__shared__ int sh[2][SCAN_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int per = (R + SCAN_THREADS - 1) / SCAN_THREADS;
	const int ra = min(R, (int)threadIdx.x * per), rb = min(R, ra + per);
	int s[2] = {0, 0};
	for (int r = ra; r < rb; r++) s[is_te[r / H] != 0] += count[r];
	int inc[2] = {s[0], s[1]};
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
		for (int k = 0; k < 2; k++) {
			int t = __shfl_up_sync(0xffffffffu, inc[k], o);
			if (lane >= o) inc[k] += t;
		}
	}
	if (lane == 31) { sh[0][warp] = inc[0]; sh[1][warp] = inc[1]; }
	__syncthreads();
	int run[2] = {inc[0] - s[0], inc[1] - s[1]};
	long long all[2] = {0, 0};
	for (int w = 0; w < SCAN_THREADS / 32; w++) {
#pragma unroll
		for (int k = 0; k < 2; k++) {
			if (w < warp) run[k] += sh[k][w];
			all[k] += sh[k][w];
		}
	}
	for (int r = ra; r < rb; r++) {
		const int k = is_te[r / H] != 0;
		(k ? off_te : off_tr)[r] = run[k];
		run[k] += count[r];
	}
	if (threadIdx.x == 0 && totals) { totals[0] = all[0]; totals[1] = all[1]; }
}

int launch_rows(int mode, float *y, const float *disp, const float *x0, const int *is_te, long rows, int H, int W, int *count,
		const int *off_tr, const int *off_te, float *nnz_tr, long long cap_tr, float *nnz_te, long long cap_te,
		cudaStream_t s)
{
	const size_t smem = (size_t)W * sizeof(float);
	const void *fn = mode == ROW_OCCLUDED ? (const void *)rows_kernel<ROW_OCCLUDED>
			 : mode == ROW_COUNT  ? (const void *)rows_kernel<ROW_COUNT>
					      : (const void *)rows_kernel<ROW_FILL>;
	if (int rc = adc_smem_optin(fn, smem)) return rc;
	if (mode == ROW_OCCLUDED)
		rows_kernel<ROW_OCCLUDED><<<(unsigned)rows, PP_THREADS, smem, s>>>(y, disp, x0, is_te, H, W, count, off_tr, off_te, nnz_tr,
									 cap_tr, nnz_te, cap_te);
	else if (mode == ROW_COUNT)
		rows_kernel<ROW_COUNT><<<(unsigned)rows, PP_THREADS, smem, s>>>(y, disp, x0, is_te, H, W, count, off_tr, off_te, nnz_tr,
								      cap_tr, nnz_te, cap_te);
	else
		rows_kernel<ROW_FILL><<<(unsigned)rows, PP_THREADS, smem, s>>>(y, disp, x0, is_te, H, W, count, off_tr, off_te, nnz_tr,
								     cap_tr, nnz_te, cap_te);
	ADC_CHECK_LAUNCH();
	return 0;
}

int check_stack(const void *a, const void *b, int n, int H, int W)
{
	if (!a || !b || n < 1 || H < 1 || W < 1) return ADCENSUS_EINVAL;
	return 0;
}

int elementwise_grid(size_t n) { return (int)std::min<size_t>((n + 255) / 256, (size_t)adc_num_sms() * 16); }

// count pass + scans into stream-ordered scratch; the offsets stay in *scratch for the fill pass (caller frees)
int count_and_scan(const float *disp, const float *x0, const int *is_te, int n, int H, int W, long long *totals, int **scratch,
		   cudaStream_t s)
{
	*scratch = nullptr;
	if (!disp || !x0 || !is_te || n < 1 || H < 1 || W < 1) return ADCENSUS_EINVAL;
	if (W > MAX_W || (size_t)n * H * W >= (1ull << 31)) return ADCENSUS_ELIMIT;
	const int R = n * H;
	int rc = adc_scratch_alloc((void **)scratch, (size_t)3 * R * sizeof(int), s);
	if (rc) return rc;
	int *count = *scratch, *off_tr = count + R, *off_te = off_tr + R;
	rc = launch_rows(ROW_COUNT, nullptr, disp, x0, is_te, R, H, W, count, nullptr, nullptr, nullptr, 0, nullptr, 0, s);
	if (rc) return rc;
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(count, is_te, R, H, off_tr, off_te, totals);
	ADC_CHECK_LAUNCH();
	return 0;
}

}  // namespace

extern "C" int adcensus_remove_nonvisible(float *y, int N, int H, int W, adcensus_stream_t stream)
{
	int rc = check_stack(y, y, N, H, W);
	if (rc) return rc;
	const size_t n = (size_t)N * H * W;
	nonvisible_kernel<<<elementwise_grid(n), 256, 0, adc_stream(stream)>>>(y, n, W);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int adcensus_remove_occluded(float *y, int N, int H, int W, adcensus_stream_t stream)
{
	int rc = check_stack(y, y, N, H, W);
	if (rc) return rc;
	if (W > MAX_W || (long)N * H >= (1l << 31)) return ADCENSUS_ELIMIT;
	return launch_rows(ROW_OCCLUDED, y, nullptr, nullptr, nullptr, (long)N * H, H, W, nullptr, nullptr, nullptr, nullptr, 0,
			   nullptr, 0, adc_stream(stream));
}

extern "C" int adcensus_remove_white(const float *x, float *y, int N, int H, int W, adcensus_stream_t stream)
{
	int rc = check_stack(x, y, N, H, W);
	if (rc) return rc;
	const size_t n = (size_t)N * H * W;
	white_kernel<<<elementwise_grid(n), 256, 0, adc_stream(stream)>>>(x, y, n);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int mccnn_kitti_nnz_count(const float *disp, const float *x0, const int *is_te, int n, int H, int W,
				     long long *counts, adcensus_stream_t stream)
{
	if (!counts) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	int *scratch = nullptr;
	int rc = count_and_scan(disp, x0, is_te, n, H, W, counts, &scratch, s);
	int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}

extern "C" int mccnn_kitti_nnz_fill(const float *disp, const float *x0, const int *is_te, int n, int H, int W,
				    float *nnz_tr, long long cap_tr, float *nnz_te, long long cap_te, adcensus_stream_t stream)
{
	if (cap_tr < 0 || cap_te < 0 || (cap_tr && !nnz_tr) || (cap_te && !nnz_te)) return ADCENSUS_EINVAL;
	if ((((uintptr_t)nnz_tr) | ((uintptr_t)nnz_te)) & 15) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	int *scratch = nullptr;
	int rc = count_and_scan(disp, x0, is_te, n, H, W, nullptr, &scratch, s);
	if (!rc) {
		const int R = n * H;
		rc = launch_rows(ROW_FILL, nullptr, disp, x0, is_te, R, H, W, nullptr, scratch + R, scratch + 2 * R, nnz_tr, cap_tr,
				 nnz_te, cap_te, s);
	}
	int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}
