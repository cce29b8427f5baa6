// rectify.cu -- undistort and rectify a calibrated stereo pair on the GPU, for sm_90a (DESIGN §22; an addition beyond the
// reference).
//
// mccnn_rectify_pair: one launch for both views, one thread per output pixel (grid-stride over H' W', blockIdx.y the view).
// Each output pixel (u, v) is mapped back to a raw source position (sx, sy) by OpenCV's initUndistortRectifyMap model, in
// fp32 with every operation rounded once (explicit __f*_rn intrinsics: no FMA contraction) and in the order the header
// states; the raw image is then sampled bilinearly with the taps clamped into the image (the border replicated), the
// weights shared by the colour channels, and the byte rint(v).  A numpy float32 restatement gives the same bytes.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;

struct View {
	const unsigned char *src;
	unsigned char *dst;
	float iR[9];                                   // inv(P[:, :3] R), row-major
	float fx, fy, cx, cy;
	float k[8];                                    // k1 k2 p1 p2 k3 k4 k5 k6
};

struct Pair {
	View v[2];
};

// the raw position (sx, sy) of output pixel (u, v); false when Z <= 0
__device__ __forceinline__ bool source_of(const View &c, float u, float v, float *sx, float *sy)
{
	const float X = __fadd_rn(__fadd_rn(__fmul_rn(c.iR[0], u), __fmul_rn(c.iR[1], v)), c.iR[2]);
	const float Y = __fadd_rn(__fadd_rn(__fmul_rn(c.iR[3], u), __fmul_rn(c.iR[4], v)), c.iR[5]);
	const float Z = __fadd_rn(__fadd_rn(__fmul_rn(c.iR[6], u), __fmul_rn(c.iR[7], v)), c.iR[8]);
	if (!(Z > 0.f)) return false;
	const float x = __fdiv_rn(X, Z), y = __fdiv_rn(Y, Z);
	const float k1 = c.k[0], k2 = c.k[1], p1 = c.k[2], p2 = c.k[3], k3 = c.k[4], k4 = c.k[5], k5 = c.k[6], k6 = c.k[7];
	const float r2 = __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y));
	const float num = __fadd_rn(1.f, __fmul_rn(r2, __fadd_rn(k1, __fmul_rn(r2, __fadd_rn(k2, __fmul_rn(r2, k3))))));
	const float den = __fadd_rn(1.f, __fmul_rn(r2, __fadd_rn(k4, __fmul_rn(r2, __fadd_rn(k5, __fmul_rn(r2, k6))))));
	const float rad = __fdiv_rn(num, den);
	const float xy2p1 = __fmul_rn(__fmul_rn(__fmul_rn(2.f, p1), x), y);
	const float xy2p2 = __fmul_rn(__fmul_rn(__fmul_rn(2.f, p2), x), y);
	const float xd = __fadd_rn(__fmul_rn(x, rad), __fadd_rn(xy2p1, __fmul_rn(p2, __fadd_rn(r2, __fmul_rn(__fmul_rn(2.f, x), x)))));
	const float yd = __fadd_rn(__fmul_rn(y, rad), __fadd_rn(__fmul_rn(p1, __fadd_rn(r2, __fmul_rn(__fmul_rn(2.f, y), y))), xy2p2));
	*sx = __fadd_rn(__fmul_rn(c.fx, xd), c.cx);
	*sy = __fadd_rn(__fmul_rn(c.fy, yd), c.cy);
	return true;
}

// floor(s) clamped into [0, n - 1], and the next tap likewise; clamped in float first, so any finite s converts safely
__device__ __forceinline__ void taps(float f, int n, int *i0, int *i1)
{
	const float hi = (float)(n - 1);
	*i0 = (int)fminf(fmaxf(f, 0.f), hi);
	*i1 = (int)fminf(fmaxf(__fadd_rn(f, 1.f), 0.f), hi);
}

__global__ void __launch_bounds__(THREADS) rectify_kernel(Pair pair, int nch, int H, int W, int Ho, int Wo,
							  unsigned char *__restrict__ valid)
{
	const View &c = pair.v[blockIdx.y];
	const long n = (long)Ho * Wo;
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		const int v = (int)(p / Wo), u = (int)(p - (long)v * Wo);
		float sx, sy;
		const bool front = source_of(c, (float)u, (float)v, &sx, &sy);
		unsigned char *out = c.dst + p * nch;
		if (!(front && isfinite(sx) && isfinite(sy))) {
			for (int ch = 0; ch < nch; ch++) out[ch] = 0;
			if (valid && blockIdx.y == 0) valid[p] = 0;
			continue;
		}
		const float fx0 = floorf(sx), fy0 = floorf(sy);
		const float a = __fsub_rn(sx, fx0), b = __fsub_rn(sy, fy0);
		const float a1 = __fsub_rn(1.f, a), b1 = __fsub_rn(1.f, b);
		int x0, x1, y0, y1;
		taps(fx0, W, &x0, &x1);
		taps(fy0, H, &y0, &y1);
		const unsigned char *r0 = c.src + (long)y0 * W * nch, *r1 = c.src + (long)y1 * W * nch;
		for (int ch = 0; ch < nch; ch++) {
			const float i00 = r0[x0 * nch + ch], i01 = r0[x1 * nch + ch];
			const float i10 = r1[x0 * nch + ch], i11 = r1[x1 * nch + ch];
			const float top = __fadd_rn(__fmul_rn(a1, i00), __fmul_rn(a, i01));
			const float bot = __fadd_rn(__fmul_rn(a1, i10), __fmul_rn(a, i11));
			out[ch] = (unsigned char)rintf(__fadd_rn(__fmul_rn(b1, top), __fmul_rn(b, bot)));
		}
		if (valid && blockIdx.y == 0)
			valid[p] = sx >= -0.5f && sx < __fsub_rn((float)W, 0.5f) && sy >= -0.5f && sy < __fsub_rn((float)H, 0.5f);
	}
}

bool overlap(const void *a, long na, const void *b, long nb)
{
	const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
	return x < y + (uintptr_t)nb && y < x + (uintptr_t)na;
}

}  // namespace

extern "C" {

int mccnn_rectify_pair(const unsigned char *left, const unsigned char *right, int nch, int H, int W, const float *params_left,
		       const float *params_right, int Ho, int Wo, unsigned char *out_left, unsigned char *out_right,
		       unsigned char *valid, adcensus_stream_t stream)
{
	if (!left || !right || !params_left || !params_right || !out_left || !out_right || (nch != 1 && nch != 3) || H < 1 ||
	    W < 1 || Ho < 1 || Wo < 1)
		return ADCENSUS_EINVAL;
	if ((long)H * W * nch >= (1l << 31) || (long)Ho * Wo * nch >= (1l << 31)) return ADCENSUS_ELIMIT;
	// no output may overlap an input or another output; the two inputs may be the same image
	const long nin = (long)H * W * nch, nout = (long)Ho * Wo * nch, nmask = (long)Ho * Wo;
	const void *bufs[5] = {left, right, out_left, out_right, valid};
	const long sizes[5] = {nin, nin, nout, nout, valid ? nmask : 0};
	for (int i = 2; i < 5; i++)
		for (int j = 0; j < i; j++)
			if (bufs[i] && overlap(bufs[i], sizes[i], bufs[j], sizes[j])) return ADCENSUS_EINVAL;
	Pair pair;
	const float *prm[2] = {params_left, params_right};
	for (int s = 0; s < 2; s++) {
		for (int k = 0; k < MCCNN_RECTIFY_NPARAM; k++)
			if (!isfinite(prm[s][k])) return ADCENSUS_EINVAL;
		View &c = pair.v[s];
		c.src = s ? right : left;
		c.dst = s ? out_right : out_left;
		for (int k = 0; k < 9; k++) c.iR[k] = prm[s][k];
		c.fx = prm[s][9];
		c.fy = prm[s][10];
		c.cx = prm[s][11];
		c.cy = prm[s][12];
		for (int k = 0; k < 8; k++) c.k[k] = prm[s][13 + k];
	}
	const long n = (long)Ho * Wo;
	const int grid = (int)std::min<long>((n + THREADS - 1) / THREADS, (long)adc_num_sms() * 8);
	rectify_kernel<<<dim3(grid, 2), THREADS, 0, adc_stream(stream)>>>(pair, nch, H, W, Ho, Wo, valid);
	ADC_CHECK_LAUNCH();
	return 0;
}

}  // extern "C"
