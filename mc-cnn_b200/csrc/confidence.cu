// confidence.cu -- a per-pixel confidence for the stereo method's disparity map, sparse maps kept by it, and the counts of
// its sparsification curve (DESIGN §19; an addition beyond the reference).
//
// Margin confidence of the final left volume V: d1 = the arg-min of argmin_pitched_kernel (first strict minimum in ascending
// d, NaN never taken, start +inf, 0 when nothing is taken) with its value c1; c2 = the minimum, by the same rule, over the d
// with |d - d1| >= 2; conf = c2 - c1 (one float rounding) when both are below +inf, else 0.  One pass over the volume keeps
// the four smallest (value, d) pairs in scan order: at most three of them lie in d1's band, so c2 is the first of the other
// ones.
//
// Sparsify and the sparsification counts order pixels by conf descending, then row-major index ascending.  Both select
// through one radix select on the 64-bit key (conf's order-preserving bits << 32 | ~index), eight 8-bit digits from the
// top: every key is distinct, so the n largest are exactly the keys >= the n-th largest.  Histograms are integer atomics
// only, so every output is exact and the same on every run.
#include "common.cuh"

namespace {

// the four smallest (value, d) pairs seen so far, in (value, d) order; d = -1: nothing taken
struct Top4 {
	float v0, v1, v2, v3;
	int d0, d1, d2, d3;
	__device__ __forceinline__ Top4()
	{
		v0 = v1 = v2 = v3 = CUDART_INF_F;
		d0 = d1 = d2 = d3 = -1;
	}
	// strict <: a later d never displaces an equal value, and NaN / +inf are never taken
	__device__ __forceinline__ void push(float v, int d)
	{
		if (!(v < v3)) return;
		if (v < v2) {
			v3 = v2; d3 = d2;
			if (v < v1) {
				v2 = v1; d2 = d1;
				if (v < v0) {
					v1 = v0; d1 = d0;
					v0 = v; d0 = d;
				} else {
					v1 = v; d1 = d;
				}
			} else {
				v2 = v; d2 = d;
			}
		} else {
			v3 = v; d3 = d;
		}
	}
	// (arg-min as main.lua:1049-1050 takes it, margin confidence)
	__device__ __forceinline__ void finish(float *disp, float *conf) const
	{
		const int a = d0 < 0 ? 0 : d0;
		float c2 = CUDART_INF_F;
		if (d1 >= 0 && abs(d1 - a) >= 2) c2 = v1;
		else if (d2 >= 0 && abs(d2 - a) >= 2) c2 = v2;
		else if (d3 >= 0 && abs(d3 - a) >= 2) c2 = v3;
		*disp = (float)a;
		*conf = (v0 < CUDART_INF_F && c2 < CUDART_INF_F) ? c2 - v0 : 0.0f;
	}
};

// argmin_pitched_kernel with the margin confidence, from the same single read of the (D, H, ld) volume
__global__ void argmin_conf_pitched_kernel(const float *__restrict__ vol, float *__restrict__ disp, float *__restrict__ conf, int D,
					   int H, int W, int ld)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
	if (x >= W) return;
	const long HW = (long)H * ld;
	const float *v = vol + (long)y * ld + x;
	Top4 t;
	int d = 0;
	for (; d + 4 <= D; d += 4) {
		float a = ld_stream(v + (long)d * HW), b = ld_stream(v + (long)(d + 1) * HW);
		float c = ld_stream(v + (long)(d + 2) * HW), e = ld_stream(v + (long)(d + 3) * HW);
		t.push(a, d);
		t.push(b, d + 1);
		t.push(c, d + 2);
		t.push(e, d + 3);
	}
	for (; d < D; d++) t.push(ld_stream(v + (long)d * HW), d);
	float dv, cv;
	t.finish(&dv, &cv);
	disp[(long)y * W + x] = dv;
	conf[(long)y * W + x] = cv;
}

// ---- radix select on (conf bits, ~index) ----

const int MAX_SEL = 20;        // the sparsification curve's 20 points
const int SEL_THREADS = 256;

struct SelState {
	unsigned long long prefix[MAX_SEL];     // the top digits of the n-th largest key found so far
	unsigned long long remaining[MAX_SEL];  // how many of the keys under `prefix` still belong to the selection
	unsigned long long M, B;                // counts: pixels with gt != 0, bad ones among them
	unsigned long long bad[MAX_SEL];
	unsigned int hist[MAX_SEL][256];
};

__device__ __forceinline__ unsigned long long sel_key(const float *conf, long i)
{
	const unsigned int u = __float_as_uint(conf[i]);
	const unsigned int o = u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);     // the bits order like the values
	return ((unsigned long long)o << 32) | (unsigned long long)(0xffffffffu - (unsigned int)i);
}

// the pixels a selection ranges over: all of them (sparsify), or gt != 0 (main.lua:1230-1236's mask)
__device__ __forceinline__ bool sel_pixel(const float *gt, long i) { return !gt || gt[i] != 0.0f; }

__device__ __forceinline__ bool is_bad(const float *pred, const float *gt, long i, float err_at)
{
	return gt[i] != 0.0f && fabsf(gt[i] - pred[i]) > err_at;
}

int sel_blocks(long n)
{
	const long b = (n + SEL_THREADS * 8 - 1) / (SEL_THREADS * 8);
	const long cap = (long)adc_num_sms() * 4;
	return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// histogram of digit `shift` / 8 of the keys that agree with each selection's prefix above it
__global__ void sel_hist_kernel(const float *__restrict__ conf, const float *__restrict__ gt, long n, int shift, int nsel, SelState *st)
{
	__shared__ unsigned int h[MAX_SEL * 256];
	__shared__ unsigned long long pre[MAX_SEL];
	for (int j = threadIdx.x; j < nsel * 256; j += blockDim.x) h[j] = 0;
	if (threadIdx.x < nsel) pre[threadIdx.x] = shift == 56 ? 0ull : st->prefix[threadIdx.x] >> (shift + 8);
	__syncthreads();
	for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
		if (!sel_pixel(gt, i)) continue;
		const unsigned long long k = sel_key(conf, i);
		const unsigned long long hi = shift == 56 ? 0ull : k >> (shift + 8);
		const unsigned int dig = (unsigned int)(k >> shift) & 255u;
		for (int s = 0; s < nsel; s++)
			if (hi == pre[s]) atomicAdd(&h[s * 256 + dig], 1u);
	}
	__syncthreads();
	for (int j = threadIdx.x; j < nsel * 256; j += blockDim.x)
		if (h[j]) atomicAdd(&st->hist[j >> 8][j & 255], h[j]);
}

// per selection: the digit under which its n-th largest key lies, from the top; clears the histogram for the next digit
__global__ void sel_pick_kernel(int shift, int nsel, SelState *st)
{
	const int s = threadIdx.x;
	if (s >= nsel) return;
	unsigned long long rem = st->remaining[s];
	if (rem) {                                     // an empty selection (n = 0) stays empty: see sel_kept
		for (int dig = 255; dig >= 0; dig--) {
			const unsigned long long c = st->hist[s][dig];
			if (c >= rem) {
				st->prefix[s] |= (unsigned long long)dig << shift;
				break;
			}
			rem -= c;
		}
		st->remaining[s] = rem;
	}
	for (int dig = 0; dig < 256; dig++) st->hist[s][dig] = 0;
}

// the selection that has kept `n` keys: remaining starts at n and stays > 0 through every digit
__device__ __forceinline__ bool sel_kept(const SelState *st, int s, unsigned long long k) { return st->remaining[s] && k >= st->prefix[s]; }

int run_select(const float *conf, const float *gt, long n, int nsel, SelState *st, cudaStream_t s)
{
	const int blocks = sel_blocks(n);
	for (int shift = 56; shift >= 0; shift -= 8) {
		sel_hist_kernel<<<blocks, SEL_THREADS, 0, s>>>(conf, gt, n, shift, nsel, st);
		ADC_CHECK_LAUNCH();
		sel_pick_kernel<<<1, 32, 0, s>>>(shift, nsel, st);
		ADC_CHECK_LAUNCH();
	}
	return 0;
}

__global__ void sparsify_init_kernel(SelState *st, long n_keep) { st->remaining[0] = (unsigned long long)n_keep; }

__global__ void sparsify_write_kernel(const float *__restrict__ disp, const float *__restrict__ conf, float *__restrict__ out, long n,
				      float invalid, const SelState *st)
{
	for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
		out[i] = sel_kept(st, 0, sel_key(conf, i)) ? disp[i] : invalid;
}

// M and B of main.lua:1228-1236
__global__ void counts_mb_kernel(const float *__restrict__ pred, const float *__restrict__ gt, long n, float err_at, SelState *st)
{
	__shared__ unsigned int m, b;
	if (threadIdx.x == 0) m = b = 0;
	__syncthreads();
	for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
		if (gt[i] != 0.0f) atomicAdd(&m, 1u);
		if (is_bad(pred, gt, i, err_at)) atomicAdd(&b, 1u);
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		atomicAdd(&st->M, (unsigned long long)m);
		atomicAdd(&st->B, (unsigned long long)b);
	}
}

// n_k = ceil(k M / 20), k = 1..20, in integers
__global__ void counts_init_kernel(SelState *st)
{
	const int s = threadIdx.x;
	if (s < MAX_SEL) st->remaining[s] = ((unsigned long long)(s + 1) * st->M + MAX_SEL - 1) / MAX_SEL;
}

__global__ void counts_bad_kernel(const float *__restrict__ pred, const float *__restrict__ conf, const float *__restrict__ gt, long n,
				  float err_at, SelState *st)
{
	__shared__ unsigned int c[MAX_SEL];
	if (threadIdx.x < MAX_SEL) c[threadIdx.x] = 0;
	__syncthreads();
	for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
		if (!is_bad(pred, gt, i, err_at)) continue;
		const unsigned long long k = sel_key(conf, i);
		for (int s = 0; s < MAX_SEL; s++)
			if (sel_kept(st, s, k)) atomicAdd(&c[s], 1u);
	}
	__syncthreads();
	if (threadIdx.x < MAX_SEL && c[threadIdx.x]) atomicAdd(&st->bad[threadIdx.x], (unsigned long long)c[threadIdx.x]);
}

__global__ void counts_out_kernel(const SelState *st, long long *counts)
{
	const int j = threadIdx.x;
	if (j == 0) counts[0] = (long long)st->M;
	if (j == 1) counts[1] = (long long)st->B;
	if (j < MAX_SEL) counts[2 + j] = (long long)st->bad[j];
}

}  // namespace

// the fused pipeline's arg-min with the confidence (csrc/pipeline.cu, direction -1)
int adc_argmin_conf_pitched(const float *vol, float *disp, float *conf, int D, int H, int W, int ld, cudaStream_t s)
{
	if (!vol || !disp || !conf || D < 1 || H < 1 || W < 1 || ld < W || H > 65535) return ADCENSUS_EINVAL;
	dim3 grid(adc_div_up(W, 128), H);
	argmin_conf_pitched_kernel<<<grid, 128, 0, s>>>(vol, disp, conf, D, H, W, ld);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" {

int mccnn_margin_confidence(const float *vol, float *disp, float *conf, int D, int H, int W, adcensus_stream_t stream)
{
	return adc_argmin_conf_pitched(vol, disp, conf, D, H, W, W, adc_stream(stream));
}

int mccnn_sparsify(const float *disp, const float *conf, float *out, int H, int W, long long n_keep, float invalid,
		   adcensus_stream_t stream)
{
	if (!disp || !conf || !out || H < 1 || W < 1) return ADCENSUS_EINVAL;
	const long n = (long)H * W;
	if (n > 0xffffffffL) return ADCENSUS_ELIMIT;
	if (n_keep < 1 || n_keep > n) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	SelState *st = nullptr;
	int rc = adc_scratch_alloc((void **)&st, sizeof(SelState), s);
	if (rc) return rc;
	rc = (int)cudaMemsetAsync(st, 0, sizeof(SelState), s);
	if (!rc) {
		sparsify_init_kernel<<<1, 1, 0, s>>>(st, n_keep);
		rc = (int)cudaPeekAtLastError();
	}
	if (!rc) rc = run_select(conf, nullptr, n, 1, st, s);
	if (!rc) {
		sparsify_write_kernel<<<sel_blocks(n), SEL_THREADS, 0, s>>>(disp, conf, out, n, invalid, st);
		rc = (int)cudaPeekAtLastError();
	}
	const int rc2 = adc_scratch_free(st, s);
	return rc ? rc : rc2;
}

int mccnn_sparsification_counts(const float *pred, const float *conf, const float *gt, int H, int W, float err_at, long long *counts,
				adcensus_stream_t stream)
{
	if (!pred || !conf || !gt || !counts || H < 1 || W < 1) return ADCENSUS_EINVAL;
	const long n = (long)H * W;
	if (n > 0xffffffffL) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	SelState *st = nullptr;
	int rc = adc_scratch_alloc((void **)&st, sizeof(SelState), s);
	if (rc) return rc;
	rc = (int)cudaMemsetAsync(st, 0, sizeof(SelState), s);
	if (!rc) {
		counts_mb_kernel<<<sel_blocks(n), SEL_THREADS, 0, s>>>(pred, gt, n, err_at, st);
		counts_init_kernel<<<1, 32, 0, s>>>(st);
		rc = (int)cudaPeekAtLastError();
	}
	if (!rc) rc = run_select(conf, gt, n, MAX_SEL, st, s);
	if (!rc) {
		counts_bad_kernel<<<sel_blocks(n), SEL_THREADS, 0, s>>>(pred, conf, gt, n, err_at, st);
		counts_out_kernel<<<1, 32, 0, s>>>(st, counts);
		rc = (int)cudaPeekAtLastError();
	}
	const int rc2 = adc_scratch_free(st, s);
	return rc ? rc : rc2;
}

}  // extern "C"
