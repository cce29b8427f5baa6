// frontend.cu -- the image front end of main.lua -a predict (frontend.make_batch, main.lua:1085-1100) and the 3-pixel error
// count of predict_kitti.lua, for sm_90a.
//
// * mccnn_frontend_batch: two decoded 8-bit views -> x_batch (2, 1, H, W), bit-identical to frontend.make_batch.  Y is
//   frontend.rgb2y's 0.299 R, + 0.587 G, + 0.114 B with every product and sum rounded separately in fp32 (numpy does not
//   contract).  frontend.standardise's three float64 sums are numpy's pairwise sums in memory order (pairwise.cuh, one tree
//   per call, both views at once): m = sum(f64 y) / n; y' = y + f32(-m) in fp32; m2 = sum(f64 y') / n;
//   var = sum((f64 y' - m2)^2) / (n - 1); out = y' / f32(sqrt(var)), an IEEE fp32 divide.
// * mccnn_kitti_error_count: dataio.bad_pixel_rate's numerator and denominator for one map against a PNG16 ground truth.
#include <algorithm>

#include "common.cuh"
#include "pairwise.cuh"

namespace {

constexpr int THREADS = 256;

// frontend.rgb2y of the interleaved pixel p, or the grey byte
template <int C>
__device__ __forceinline__ float luma(const unsigned char *v, long p)
{
	if (C == 1) return (float)v[p];
	const unsigned char *px = v + 3 * p;
	const float y = __fadd_rn(__fmul_rn(0.299f, (float)px[0]), __fmul_rn(0.587f, (float)px[1]));
	return __fadd_rn(y, __fmul_rn(0.114f, (float)px[2]));
}

// per view: stats[3 view] = m, [3 view + 1] = m2, [3 view + 2] = var
__device__ __forceinline__ float neg_mean(const double *stats, int view) { return (float)(-stats[3 * view]); }

// the terms of standardise's float64 sums: PASS 0 f64(y), 1 f64(y + f32(-m)), 2 (f64(y + f32(-m)) - m2)^2
template <int C, int PASS>
struct Term {
	const unsigned char *left, *right;
	const double *stats;
	__device__ double operator()(int view, long p) const
	{
		const float y = luma<C>(view ? right : left, p);
		if (PASS == 0) return (double)y;
		const double x = (double)__fadd_rn(y, neg_mean(stats, view));
		if (PASS == 1) return x;
		const double d = __dsub_rn(x, stats[3 * view + 1]);
		return __dmul_rn(d, d);
	}
};

// stats[3 view + k] = sum / div (k = 0, 1: div = n; k = 2: div = n - 1)
struct Quotient {
	double *stats;
	int k;
	double div;
	__device__ void operator()(int view, double sum) const { stats[3 * view + k] = __ddiv_rn(sum, div); }
};

template <int C>
__global__ void normalise_kernel(const unsigned char *__restrict__ left, const unsigned char *__restrict__ right,
				 const double *__restrict__ stats, long hw, float *__restrict__ out)
{
	const int view = blockIdx.y;
	const unsigned char *v = view ? right : left;
	const float negm = neg_mean(stats, view), sd = (float)__dsqrt_rn(stats[3 * view + 2]);
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x)
		out[view * hw + p] = __fdiv_rn(__fadd_rn(luma<C>(v, p), negm), sd);
}

template <int C>
int frontend_batch(const unsigned char *left, const unsigned char *right, long hw, float *out, double *stats, cudaStream_t s)
{
	pairwise::Sum<double> t;
	int rc = t.init(hw, 2, s);
	if (!rc) rc = t.sum(Term<C, 0>{left, right, stats}, Quotient{stats, 0, (double)hw});
	if (!rc) rc = t.sum(Term<C, 1>{left, right, stats}, Quotient{stats, 1, (double)hw});
	if (!rc) rc = t.sum(Term<C, 2>{left, right, stats}, Quotient{stats, 2, (double)(hw - 1)});
	if (!rc) {
		const dim3 grid((unsigned)std::min<long>((hw + THREADS - 1) / THREADS, (long)adc_num_sms() * 8), 2);
		normalise_kernel<C><<<grid, THREADS, 0, s>>>(left, right, stats, hw, out);
		rc = (int)cudaPeekAtLastError();
	}
	const int rf = t.release();
	return rc ? rc : rf;
}

// counts[0] += #(gt != 0 and |gt / 256 - disp| > err_at), counts[1] += #(gt != 0); fp32 as numpy evaluates it
__global__ void error_count_kernel(const float *__restrict__ disp, const unsigned short *__restrict__ gt, long n, float err_at,
				   unsigned long long *__restrict__ counts)
{
	unsigned bad = 0, valid = 0;
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		const unsigned g = gt[p];
		if (g) {
			valid++;
			const float actual = __fmul_rn((float)g, 1.f / 256.f);      // read_png16's v / 256, exact
			bad += fabsf(__fsub_rn(actual, disp[p])) > err_at;          // NaN is not > err_at
		}
	}
#pragma unroll
	for (int o = 16; o; o >>= 1) {
		bad += __shfl_xor_sync(0xffffffffu, bad, o);
		valid += __shfl_xor_sync(0xffffffffu, valid, o);
	}
	if ((threadIdx.x & 31) == 0 && valid) {
		atomicAdd(counts, (unsigned long long)bad);
		atomicAdd(counts + 1, (unsigned long long)valid);
	}
}

}  // namespace

extern "C" int mccnn_frontend_batch(const unsigned char *left, const unsigned char *right, int nch, int H, int W, float *x_batch,
				    double *stats, adcensus_stream_t stream)
{
	if (!left || !right || !x_batch || !stats || (nch != 1 && nch != 3) || H < 1 || W < 1 || (long)H * W < 2)
		return ADCENSUS_EINVAL;
	if ((long)H * W * nch >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	const long hw = (long)H * W;
	return nch == 1 ? frontend_batch<1>(left, right, hw, x_batch, stats, s) : frontend_batch<3>(left, right, hw, x_batch, stats, s);
}

extern "C" int mccnn_kitti_error_count(const float *disp, const unsigned short *gt, int H, int W, float err_at, long long *counts,
				       adcensus_stream_t stream)
{
	if (!disp || !gt || !counts || H < 1 || W < 1 || !(err_at >= 0.f)) return ADCENSUS_EINVAL;
	if ((long)H * W >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	cudaError_t e = cudaMemsetAsync(counts, 0, 2 * sizeof(long long), s);
	if (e != cudaSuccess) return (int)e;
	const long n = (long)H * W;
	const int grid = (int)std::min<long>((n + THREADS - 1) / THREADS, (long)adc_num_sms() * 8);
	error_count_kernel<<<grid, THREADS, 0, s>>>(disp, gt, n, err_at, (unsigned long long *)counts);
	ADC_CHECK_LAUNCH();
	return 0;
}
