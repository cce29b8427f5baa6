// preprocess_mb.cu -- the per-pixel work of preprocess_mb.py (Middlebury 2014/2006/2005/2003/2001 and MiddEval3), for sm_90a.
//
// * mccnn_mb_views: read_im (preprocess_mb.py:85-97) from decoded bytes -- cv2's BGR2GRAY (or the RGB planes), then
//   (x - x.mean()) / x.std() exactly as numpy computes it in float32: numpy's pairwise sum over the array in memory order
//   (pixels, channels interleaved for rgb), the two quotients by the element count in float64 rounded to float32 (numpy
//   divides a float32 by an intp), a float32 sqrt and IEEE float32 subtraction and division.  One thread per leaf of the
//   pairwise tree (<= 128 elements), then the fixed combine tree, one block per view (pairwise.cuh): deterministic,
//   bit-identical.
// * mccnn_mb_half_image: `convert X -resize 50%` restated (Lanczos-3, renormalised at the border, fp32, rounded half up).
//   ImageMagick is not pinned: this is a restatement of its documented filter, not a bit-for-bit copy.
// * mccnn_mb_half_disp: load_pfm(.., True) (:13-26): x / 2, then the second smallest of each 2x2 block in np.sort order.
// * mccnn_mb_mask: `computemask disp0 [disp0y] disp1 -1` restated (the MiddEval3 SDK is not pinned either); arithmetic in
//   fp64 so that the rule is exact for float32 maps.
// * mccnn_mb_nnz_count / _fill: dispnoc (disp0 where mask == 255, else 0) and the rows (image, y, x, disp0) of every
//   mask == 255 pixel in row-major order (:177-182), sized by a count pass.
// DESIGN.md has the exactness arguments.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "pairwise.cuh"

namespace {

constexpr int ROW_THREADS = 256;
constexpr int ROW_WARPS = ROW_THREADS / 32;
constexpr int SCAN_THREADS = 1024;
constexpr int TAPS = 12;                  // Lanczos-3 at scale 1/2: source pixels 2x-5 .. 2x+6

// ---- views --------------------------------------------------------------------------------------------------------

// cv2.cvtColor(float32 BGR, COLOR_BGR2GRAY) of OpenCV 4.x, evaluated as fma(R, .299, fma(B, .114, G * .587))
__device__ __forceinline__ float grey_of(const unsigned char *px)
{
	const float r = px[0], g = px[1], b = px[2];
	return __fmaf_rn(r, 0.299f, __fmaf_rn(b, 0.114f, __fmul_rn(g, 0.587f)));
}

// element i of the view in numpy's memory order, minus m and squared when SQUARE (the x - mean, x * x of np.std)
template <int C, bool SQUARE>
__device__ __forceinline__ float element(const unsigned char *v, long i, float m)
{
	const float x = C == 1 ? grey_of(v + 3 * i) : (float)v[i];
	if (!SQUARE) return x;
	const float d = __fsub_rn(x, m);
	return __fmul_rn(d, d);
}

// element i of view `view` minus its mean and squared when SQUARE: the terms of np.mean / np.std's pairwise sums
template <int C, bool SQUARE>
struct ViewElem {
	const unsigned char *rgb;
	long view_bytes;
	const float *stats;
	__device__ float operator()(int view, long i) const
	{
		return element<C, SQUARE>(rgb + view * view_bytes, i, SQUARE ? stats[2 * view] : 0.f);
	}
};

// stats[2 view] = the mean, or stats[2 view + 1] = the std when SQUARE: the sum / count in float64 rounded to float32 (numpy
// divides a float32 by an intp), then a float32 sqrt
template <bool SQUARE>
struct ViewFinish {
	float *stats;
	long count;
	__device__ void operator()(int view, float sum) const
	{
		const float s = (float)((double)sum / (double)count);
		if (SQUARE)
			stats[2 * view + 1] = __fsqrt_rn(s);
		else
			stats[2 * view] = s;
	}
};

template <int C>
__global__ void normalise_kernel(const unsigned char *__restrict__ rgb, float *__restrict__ out, const float *__restrict__ stats,
				 long hw)
{
	const int view = blockIdx.y;
	const float m = stats[2 * view], s = stats[2 * view + 1];
	const unsigned char *v = rgb + (long)view * hw * 3;
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x) {
#pragma unroll
		for (int c = 0; c < C; c++) {
			const float x = C == 1 ? grey_of(v + 3 * p) : (float)v[3 * p + c];
			out[((long)view * C + c) * hw + p] = __fdiv_rn(__fsub_rn(x, m), s);
		}
	}
}

template <int C>
int pairwise_stats(const unsigned char *rgb, int n, long hw, float *stats, cudaStream_t s)
{
	const long count = hw * C, view_bytes = hw * 3;
	pairwise::Sum<float> t;
	int rc = t.init(count, n, s);
	if (!rc) rc = t.sum(ViewElem<C, false>{rgb, view_bytes, stats}, ViewFinish<false>{stats, count});
	if (!rc) rc = t.sum(ViewElem<C, true>{rgb, view_bytes, stats}, ViewFinish<true>{stats, count});
	const int rf = t.release();
	return rc ? rc : rf;
}

// ---- halving ------------------------------------------------------------------------------------------------------

struct Taps {
	float w[TAPS];
};

// one pass of the separable filter along one axis: out[o] = sum_k w[k] src[2o - 5 + k] / sum_k w[k] over the taps inside
// [0, len); `stride` steps along the filtered axis, the other coordinates are folded into `base`
__device__ __forceinline__ float lanczos_tap_sum(const Taps &t, int o, int len, long stride, long base, const float *f,
						  const unsigned char *b)
{
	float acc = 0.f, ws = 0.f;
#pragma unroll
	for (int k = 0; k < TAPS; k++) {
		const int j = 2 * o - 5 + k;
		if (j < 0 || j >= len) continue;
		const float v = f ? f[base + j * stride] : (float)b[base + j * stride];
		acc = __fmaf_rn(t.w[k], v, acc);
		ws = __fadd_rn(ws, t.w[k]);
	}
	return __fdiv_rn(acc, ws);
}

// (n, H, W, 3) bytes -> (n, H, W/2, 3) float
__global__ void half_rows_kernel(const unsigned char *__restrict__ in, float *__restrict__ tmp, int n, int H, int W, Taps t)
{
	const int Wo = W / 2;
	const long total = (long)n * H * Wo * 3;
	for (long id = (long)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (long)gridDim.x * blockDim.x) {
		const int c = (int)(id % 3);
		const int x = (int)(id / 3 % Wo);
		const long row = id / (3l * Wo);                                   // view * H + y
		tmp[id] = lanczos_tap_sum(t, x, W, 3, row * W * 3 + c, nullptr, in);
	}
}

// (n, H, W/2, 3) float -> (n, H/2, W/2, 3) bytes, rounded half up and clamped
__global__ void half_cols_kernel(const float *__restrict__ tmp, unsigned char *__restrict__ out, int n, int H, int W, Taps t)
{
	const int Wo = W / 2, Ho = H / 2;
	const long total = (long)n * Ho * Wo * 3;
	for (long id = (long)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (long)gridDim.x * blockDim.x) {
		const long cx = id % (3l * Wo);                                    // x * 3 + c
		const int y = (int)(id / (3l * Wo) % Ho);
		const long view = id / (3l * Wo * Ho);
		const float v = lanczos_tap_sum(t, y, H, 3l * Wo, view * H * Wo * 3 + cx, tmp, nullptr);
		out[id] = (unsigned char)fminf(255.f, fmaxf(0.f, floorf(v + 0.5f)));
	}
}

// np.sort's order: -inf < finite < +inf < NaN
__device__ __forceinline__ bool sort_less(float a, float b) { return a < b || (!isnan(a) && isnan(b)); }

__global__ void half_disp_kernel(const float *__restrict__ in, float *__restrict__ out, int n, int H, int W)
{
	const int Ho = H / 2, Wo = W / 2;
	const long total = (long)n * Ho * Wo;
	for (long id = (long)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (long)gridDim.x * blockDim.x) {
		const int x = (int)(id % Wo), y = (int)(id / Wo % Ho);
		const long base = (id / ((long)Wo * Ho) * H + 2 * y) * (long)W + 2 * x;
		float v[4] = {__fdiv_rn(in[base], 2.f), __fdiv_rn(in[base + 1], 2.f), __fdiv_rn(in[base + W], 2.f),
			      __fdiv_rn(in[base + W + 1], 2.f)};
		// second smallest: the smaller of (max of the lower pair, min of the upper pair) after one compare-exchange each
		auto cx = [](float &a, float &b) {
			if (sort_less(b, a)) { float t = a; a = b; b = t; }
		};
		cx(v[0], v[1]);
		cx(v[2], v[3]);
		cx(v[0], v[2]);                                                    // v[0] = smallest
		cx(v[1], v[3]);                                                    // v[3] = largest
		cx(v[1], v[2]);                                                    // v[1] = second smallest
		out[id] = v[1];
	}
}

// ---- mask and lists -----------------------------------------------------------------------------------------------

__global__ void mask_kernel(const float *__restrict__ d0, const float *__restrict__ dy, const float *__restrict__ d1, int H,
			    int W, unsigned char *__restrict__ mask)
{
	const long total = (long)H * W;
	for (long id = (long)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (long)gridDim.x * blockDim.x) {
		const int x = (int)(id % W), y = (int)(id / W);
		const double d = d0[id];
		unsigned char m;
		if (!isfinite(d)) {
			m = 0;
		} else {
			const double v = dy ? (double)dy[id] : 0.0;
			const double fx = floor((double)x - d + 0.5), fy = floor((double)y + v + 0.5);
			if (!(fx >= 0 && fx < W && fy >= 0 && fy < H)) {             // a non-finite disp0y is out of frame
				m = 128;
			} else {
				const double r = d1[(long)fy * W + (long)fx];
				m = fabs(d - r) <= 1.0 ? 255 : 128;                  // inf or NaN on the right side fails
			}
		}
		mask[id] = m;
	}
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
	for (int w = 0; w < ROW_WARPS; w++) {
		if (w < warp) base += sh[w];
		all += sh[w];
	}
	__syncthreads();
	*total = all;
	return base + inc - v;
}

// One block per row.  FILL = false: count[y] = the row's mask == 255 pixels.  FILL = true: dispnoc row and the rows
// (image, y, x, d0) at off[y] in ascending x.
template <bool FILL>
__global__ void __launch_bounds__(ROW_THREADS) rows_kernel(const float *__restrict__ d0, const unsigned char *__restrict__ mask,
							   int W, int *__restrict__ count, const int *__restrict__ off, float image,
							   float *__restrict__ dispnoc, float *__restrict__ nnz, long long cap)
{
	__shared__ int shi[ROW_WARPS];
	const int y = blockIdx.x;
	const long base = (long)y * W;
	const int per = (W + ROW_THREADS - 1) / ROW_THREADS;
	const int xa = min(W, (int)threadIdx.x * per), xb = min(W, xa + per);
	int c = 0;
	for (int x = xa; x < xb; x++) c += mask[base + x] == 255;
	int total = 0;
	const int before = block_prefix_sum_exclusive(c, shi, &total);
	if (!FILL) {
		if (threadIdx.x == 0) count[y] = total;
		return;
	}
	long long t = (long long)off[y] + before;
	for (int x = xa; x < xb; x++) {
		const bool keep = mask[base + x] == 255;
		const float d = keep ? d0[base + x] : 0.f;
		dispnoc[base + x] = d;
		if (keep) {
			if (t < cap) *reinterpret_cast<float4 *>(nnz + 4 * t) = make_float4(image, (float)y, (float)x, d);
			t++;
		}
	}
}

// exclusive scan of count[0..R) into off, *total = the sum; one block
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const int *__restrict__ count, int R, int *__restrict__ off,
							    long long *__restrict__ total)
{
	__shared__ int sh[SCAN_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int per = (R + SCAN_THREADS - 1) / SCAN_THREADS;
	const int ra = min(R, (int)threadIdx.x * per), rb = min(R, ra + per);
	int s = 0;
	for (int r = ra; r < rb; r++) s += count[r];
	int inc = s;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		int t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= o) inc += t;
	}
	if (lane == 31) sh[warp] = inc;
	__syncthreads();
	int run = inc - s;
	long long all = 0;
	for (int w = 0; w < SCAN_THREADS / 32; w++) {
		if (w < warp) run += sh[w];
		all += sh[w];
	}
	for (int r = ra; r < rb; r++) {
		off[r] = run;
		run += count[r];
	}
	if (threadIdx.x == 0 && total) *total = all;
}

int elementwise_grid(long n) { return (int)std::min<long>((n + 255) / 256, (long)adc_num_sms() * 16); }

bool frame_ok(int H, int W) { return H >= 1 && W >= 1 && (long)H * W < (1l << 31); }

// count pass + scan into stream-ordered scratch (2 H ints: counts, offsets; the caller frees)
int count_and_scan(const unsigned char *mask, int H, int W, long long *total, int **scratch, cudaStream_t s)
{
	*scratch = nullptr;
	if (!mask || !frame_ok(H, W)) return ADCENSUS_EINVAL;
	int rc = adc_scratch_alloc((void **)scratch, (size_t)2 * H * sizeof(int), s);
	if (rc) return rc;
	int *count = *scratch, *off = count + H;
	rows_kernel<false><<<H, ROW_THREADS, 0, s>>>(nullptr, mask, W, count, nullptr, 0.f, nullptr, nullptr, 0);
	ADC_CHECK_LAUNCH();
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(count, H, off, total);
	ADC_CHECK_LAUNCH();
	return 0;
}

Taps lanczos_taps()
{
	// L(t) = sinc(t) sinc(t / 3) at t = (k - 5.5) / 2 (source pixel centre j + 0.5 against output centre 2x + 1, in output
	// pixels), in double, rounded to float
	Taps t;
	const double pi = 3.14159265358979323846;
	for (int k = 0; k < TAPS; k++) {
		const double u = (k - 5.5) / 2;
		t.w[k] = (float)(sin(pi * u) / (pi * u) * (sin(pi * u / 3) / (pi * u / 3)));
	}
	return t;
}

}  // namespace

extern "C" int mccnn_mb_views(const unsigned char *rgb, float *out, int n, int H, int W, int nchannel, adcensus_stream_t stream)
{
	if (!rgb || !out || n < 1 || n > 65535 || !frame_ok(H, W) || (nchannel != 1 && nchannel != 3)) return ADCENSUS_EINVAL;
	if ((long)H * W * 3 >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	const long hw = (long)H * W;
	float *stats = nullptr;
	int rc = adc_scratch_alloc((void **)&stats, sizeof(float) * 2 * n, s);
	if (rc) return rc;
	rc = nchannel == 1 ? pairwise_stats<1>(rgb, n, hw, stats, s) : pairwise_stats<3>(rgb, n, hw, stats, s);
	if (!rc) {
		const dim3 grid((unsigned)std::min<long>((hw + 255) / 256, 4096), n);
		if (nchannel == 1)
			normalise_kernel<1><<<grid, 256, 0, s>>>(rgb, out, stats, hw);
		else
			normalise_kernel<3><<<grid, 256, 0, s>>>(rgb, out, stats, hw);
		cudaError_t e = cudaPeekAtLastError();
		if (e != cudaSuccess) rc = (int)e;
	}
	int rf = adc_scratch_free(stats, s);
	return rc ? rc : rf;
}

extern "C" int mccnn_mb_half_image(const unsigned char *in, unsigned char *out, int n, int H, int W, adcensus_stream_t stream)
{
	if (!in || !out || n < 1 || !frame_ok(H, W) || H % 2 || W % 2) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	float *tmp = nullptr;
	int rc = adc_scratch_alloc((void **)&tmp, sizeof(float) * (size_t)n * H * (W / 2) * 3, s);
	if (rc) return rc;
	const Taps t = lanczos_taps();
	half_rows_kernel<<<elementwise_grid((long)n * H * (W / 2) * 3), 256, 0, s>>>(in, tmp, n, H, W, t);
	cudaError_t e = cudaPeekAtLastError();
	if (e == cudaSuccess) {
		half_cols_kernel<<<elementwise_grid((long)n * (H / 2) * (W / 2) * 3), 256, 0, s>>>(tmp, out, n, H, W, t);
		e = cudaPeekAtLastError();
	}
	int rf = adc_scratch_free(tmp, s);
	return e != cudaSuccess ? (int)e : rf;
}

extern "C" int mccnn_mb_half_disp(const float *in, float *out, int n, int H, int W, adcensus_stream_t stream)
{
	if (!in || !out || n < 1 || !frame_ok(H, W) || H % 2 || W % 2) return ADCENSUS_EINVAL;
	const long total = (long)n * (H / 2) * (W / 2);
	half_disp_kernel<<<elementwise_grid(total), 256, 0, adc_stream(stream)>>>(in, out, n, H, W);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int mccnn_mb_mask(const float *d0, const float *d0y, const float *d1, int H, int W, unsigned char *mask,
			     adcensus_stream_t stream)
{
	if (!d0 || !d1 || !mask || !frame_ok(H, W)) return ADCENSUS_EINVAL;
	mask_kernel<<<elementwise_grid((long)H * W), 256, 0, adc_stream(stream)>>>(d0, d0y, d1, H, W, mask);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int mccnn_mb_nnz_count(const unsigned char *mask, int H, int W, long long *count, adcensus_stream_t stream)
{
	if (!count) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	int *scratch = nullptr;
	int rc = count_and_scan(mask, H, W, count, &scratch, s);
	int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}

extern "C" int mccnn_mb_nnz_fill(const float *d0, const unsigned char *mask, int H, int W, int image, float *dispnoc, float *nnz,
				 long long cap, adcensus_stream_t stream)
{
	if (!d0 || !dispnoc || cap < 0 || (cap && !nnz) || ((uintptr_t)nnz & 15) || image < 1 || image > (1 << 24))
		return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	int *scratch = nullptr;
	int rc = count_and_scan(mask, H, W, nullptr, &scratch, s);
	if (!rc) {
		rows_kernel<true><<<H, ROW_THREADS, 0, s>>>(d0, mask, W, nullptr, scratch + H, (float)image, dispnoc, nnz, cap);
		cudaError_t e = cudaPeekAtLastError();
		if (e != cudaSuccess) rc = (int)e;
	}
	int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}
