// track.cu -- frame-to-model tracking against the distance field, for sm_90a (DESIGN §25; an addition beyond the
// reference).
//
// A handle owns two three-level pyramids at one (H, W): the source (a new frame's disparity) and the model (the depth
// TSDF.render returns at the previous pose).  Level l keeps the full-resolution pixels (2^l x, 2^l y); each level holds
// float64 vertex and normal planes, NaN where there is none.  mccnn_track_step runs one projective point-to-plane ICP
// reduce: each source pixel's 28 float64 terms (the upper triangle of J^T J, J^T r, r^2) are summed in a fixed tree --
// chunks of 1024 pixels in row-major order, stride halving inside each chunk, then the same over the chunk sums padded to
// a power of two -- so the sums have the same bits on every run and GPU and can be restated in numpy.  The inlier count is
// an integer, summed by atomics.  One device-to-host copy per step returns the sums and the counts.
//
// The photometric term (DESIGN §26): intensity pyramids of the frame's left image and of the previous frame's (with its
// gradients), allocated on first use; given gates, the same step kernel reduces each pixel's photometric terms after its
// geometric ones, through the same tree and shared buffer, in one pass and one read-back.
#include <math.h>

#include "camera.cuh"

namespace {

constexpr int LEVELS = MCCNN_TRACK_LEVELS;
constexpr int NS = MCCNN_TRACK_SUMS;              // 21 + 6 + 1
constexpr int CH = 1024;                          // pixels per chunk
constexpr int RT = 256;                           // threads per chunk: 4 pixels each
constexpr int RED = 1024;                         // threads of the chunk-sum reduction

__device__ __forceinline__ double dnan() { return __longlong_as_double(0x7ff8000000000000ll); }

struct Maps {
	double *v[3], *n[3];                          // x, y, z planes of the vertices and the normals
};

Maps maps_at(double *base, long long np)
{
	Maps m;
	for (int a = 0; a < 3; a++) {
		m.v[a] = base + a * np;
		m.n[a] = base + (3 + a) * np;
	}
	return m;
}

// a level's vertex from the full-resolution pixel (2^l x, 2^l y): of its disparity by §20's rule (source), or of the
// rendered depth, NaN = none (model); fp32 camera.cuh bits promoted to float64.  `nvert` counts the source's vertices.
__global__ void __launch_bounds__(256) vertex_kernel(const float *__restrict__ src, int is_depth, int W, int l, int hl, int wl,
						     Cam c, Maps m, unsigned long long *__restrict__ nvert)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	const long long np = (long long)hl * wl;
	bool ok = false;
	if (i < np) {
		const int x = (int)(i % wl) << l, y = (int)(i / wl) << l;
		const float s = src[(long long)y * W + x];
		float z = s;
		ok = is_depth ? !isnan(s) : depth_of(s, c, &z);
		m.v[0][i] = ok ? (double)lateral(x, c.cx, z, c.f) : dnan();
		m.v[1][i] = ok ? (double)lateral(y, c.cy, z, c.f) : dnan();
		m.v[2][i] = ok ? (double)z : dnan();
	}
	const int k = __syncthreads_count(ok);
	if (nvert && threadIdx.x == 0 && k) atomicAdd(nvert, (unsigned long long)k);
}

// n = (V(x+1, y) - V(x, y)) x (V(x, y+1) - V(x, y)), normalised, flipped to face the camera; NaN when a vertex is missing
// or |n| is 0 or not finite.  float64, each operation rounded once, no FMA.
__global__ void __launch_bounds__(256) normal_kernel(int hl, int wl, Maps m)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (long long)hl * wl) return;
	const int x = (int)(i % wl), y = (int)(i / wl);
	double n[3] = {dnan(), dnan(), dnan()};
	if (x + 1 < wl && y + 1 < hl && !isnan(m.v[0][i]) && !isnan(m.v[0][i + 1]) && !isnan(m.v[0][i + wl])) {
		double p[3], a[3], b[3];
		for (int k = 0; k < 3; k++) {
			p[k] = m.v[k][i];
			a[k] = __dsub_rn(m.v[k][i + 1], p[k]);
			b[k] = __dsub_rn(m.v[k][i + wl], p[k]);
		}
		const double c0 = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
		const double c1 = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
		const double c2 = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
		const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(c0, c0), __dmul_rn(c1, c1)), __dmul_rn(c2, c2)));
		if (len > 0.0 && len <= 1.7976931348623157e308) {
			n[0] = __ddiv_rn(c0, len);
			n[1] = __ddiv_rn(c1, len);
			n[2] = __ddiv_rn(c2, len);
			const double dot = __dadd_rn(__dadd_rn(__dmul_rn(n[0], p[0]), __dmul_rn(n[1], p[1])), __dmul_rn(n[2], p[2]));
			if (dot > 0.0)
				for (int k = 0; k < 3; k++) n[k] = -n[k];
		}
	}
	for (int k = 0; k < 3; k++) m.n[k][i] = n[k];
}

struct Step {
	int hl, wl;
	double f, cx, cy, scale;                     // the model camera, and 2^-l
	double d2, cos_t;                            // delta^2, cos(theta)
};

// pixel i's Jacobian row J and residual r (zero, and false, when the pixel is skipped)
__device__ __forceinline__ bool pixel_term(long long i, const Maps &S, const Maps &M, const Pose &T, const Step &st, double *J)
{
	for (int k = 0; k < 7; k++) J[k] = 0.0;
	if (i >= (long long)st.hl * st.wl) return false;
	const double n0 = S.n[0][i];
	if (isnan(n0)) return false;                 // no source normal (and so no source vertex)
	double q[3], ns[3];
	to_world(S.v[0][i], S.v[1][i], S.v[2][i], T, q);
	const double *r = T.r;
	for (int a = 0; a < 3; a++)
		ns[a] = __dadd_rn(__dadd_rn(__dmul_rn(r[4 * a], n0), __dmul_rn(r[4 * a + 1], S.n[1][i])), __dmul_rn(r[4 * a + 2], S.n[2][i]));
	if (!(q[2] > 0.0)) return false;
	const double u = floor(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[0], q[2]), st.f), st.cx), st.scale), 0.5));
	const double v = floor(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[1], q[2]), st.f), st.cy), st.scale), 0.5));
	if (!(u >= 0.0 && u < st.wl && v >= 0.0 && v < st.hl)) return false;
	const long long j = (long long)v * st.wl + (long long)u;
	const double nm[3] = {M.n[0][j], M.n[1][j], M.n[2][j]};
	if (isnan(nm[0])) return false;              // no model normal (and so no model vertex)
	const double d[3] = {__dsub_rn(q[0], M.v[0][j]), __dsub_rn(q[1], M.v[1][j]), __dsub_rn(q[2], M.v[2][j])};
	const double dd = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
	const double c = __dadd_rn(__dadd_rn(__dmul_rn(ns[0], nm[0]), __dmul_rn(ns[1], nm[1])), __dmul_rn(ns[2], nm[2]));
	if (!(dd <= st.d2 && c >= st.cos_t)) return false;
	J[0] = __dsub_rn(__dmul_rn(q[1], nm[2]), __dmul_rn(q[2], nm[1]));
	J[1] = __dsub_rn(__dmul_rn(q[2], nm[0]), __dmul_rn(q[0], nm[2]));
	J[2] = __dsub_rn(__dmul_rn(q[0], nm[1]), __dmul_rn(q[1], nm[0]));
	J[3] = nm[0];
	J[4] = nm[1];
	J[5] = nm[2];
	J[6] = __dadd_rn(__dadd_rn(__dmul_rn(nm[0], d[0]), __dmul_rn(nm[1], d[1])), __dmul_rn(nm[2], d[2]));
	return true;
}

// the first two halvings of the four pixels' term J_a J_b (J[6] is r): (P0 + P2) + (P1 + P3), pixel p at t + 256 p
__device__ __forceinline__ double quad(const double (*J)[7], int a, int b)
{
	return __dadd_rn(__dadd_rn(__dmul_rn(J[0][a], J[0][b]), __dmul_rn(J[2][a], J[2][b])),
			 __dadd_rn(__dmul_rn(J[1][a], J[1][b]), __dmul_rn(J[3][a], J[3][b])));
}

// the tree over the four pixels' terms of each thread (pixel p at t + 256 p): the first two halvings in registers
// ((a_t + a_t+512) + (a_t+256 + a_t+768)), strides 128, 64 and 32 through the shared buffer sh, 16 .. 1 through warp
// shuffles; the chunk's 28 sums to part[k P + chunk]
__device__ __forceinline__ void reduce_chunk(const double (*J)[7], double *sh, double *__restrict__ part, int P)
{
	double s[NS];
	{
		int k = 0;
#pragma unroll
		for (int a = 0; a < 6; a++)
#pragma unroll
			for (int b = a; b < 6; b++, k++) s[k] = quad(J, a, b);
#pragma unroll
		for (int a = 0; a < 6; a++) s[21 + a] = quad(J, a, 6);
		s[27] = quad(J, 6, 6);
	}
#pragma unroll
	for (int stride = 128; stride >= 32; stride >>= 1) {
		const int t = threadIdx.x;
		if (t >= stride && t < 2 * stride)
#pragma unroll
			for (int k = 0; k < NS; k++) sh[k * stride + t - stride] = s[k];
		__syncthreads();
		if (t < stride)
#pragma unroll
			for (int k = 0; k < NS; k++) s[k] = __dadd_rn(s[k], sh[k * stride + t]);
		__syncthreads();
	}
	if (threadIdx.x < 32) {
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1)
#pragma unroll
			for (int k = 0; k < NS; k++) s[k] = __dadd_rn(s[k], __shfl_down_sync(0xffffffffu, s[k], off));
		if (threadIdx.x == 0)
#pragma unroll
			for (int k = 0; k < NS; k++) part[(long long)k * P + blockIdx.x] = s[k];
	}
}

// ---- the photometric term (DESIGN §26) ----

// level 0 of an intensity pyramid: the byte, or ((R + G) + B) / 3, in fp32
__global__ void __launch_bounds__(256) grey_kernel(const unsigned char *__restrict__ img, int nch, long long np, float *__restrict__ I)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= np) return;
	if (nch == 1) {
		I[i] = (float)img[i];
	} else {
		const unsigned char *p = img + 3 * i;
		I[i] = __fdiv_rn(__fadd_rn(__fadd_rn((float)p[0], (float)p[1]), (float)p[2]), 3.0f);
	}
}

// (L(a - 1) / 4 + L(a) / 2) + L(a + 1) / 4 along a row (step 1) or a column (step w) of level L, indices clamped to [0, n)
__device__ __forceinline__ float blur3(const float *L, int a, int n, long long step)
{
	const float l = L[(long long)max(a - 1, 0) * step], c = L[(long long)a * step], r = L[(long long)min(a + 1, n - 1) * step];
	return __fadd_rn(__fadd_rn(__fmul_rn(0.25f, l), __fmul_rn(0.5f, c)), __fmul_rn(0.25f, r));
}

// level l + 1 (h2 x w2) of level l (h x w): the [1/4 1/2 1/4] blur at even pixels, the three rows' blurs first
__global__ void __launch_bounds__(256) down_kernel(const float *__restrict__ L, int h, int w, float *__restrict__ out, int h2, int w2)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (long long)h2 * w2) return;
	const int x = 2 * (int)(i % w2), y = 2 * (int)(i / w2);
	float r[3];
#pragma unroll
	for (int k = 0; k < 3; k++) r[k] = blur3(L + (long long)min(max(y - 1 + k, 0), h - 1) * w, x, w, 1);
	out[i] = __fadd_rn(__fadd_rn(__fmul_rn(0.25f, r[0]), __fmul_rn(0.5f, r[1])), __fmul_rn(0.25f, r[2]));
}

// central differences 0.5 (L(x + 1) - L(x - 1)) in float64, NaN on the level's border
__global__ void __launch_bounds__(256) gradient_kernel(const float *__restrict__ L, int h, int w, double *__restrict__ gx,
						       double *__restrict__ gy)
{
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (long long)h * w) return;
	const int x = (int)(i % w), y = (int)(i / w);
	gx[i] = x >= 1 && x + 1 < w ? __dmul_rn(0.5, __dsub_rn((double)L[i + 1], (double)L[i - 1])) : dnan();
	gy[i] = y >= 1 && y + 1 < h ? __dmul_rn(0.5, __dsub_rn((double)L[i + w], (double)L[i - w])) : dnan();
}

struct Photo {
	const float *Is, *Ir;                        // the level's source and reference intensities
	const double *gx, *gy;                       // the reference's gradients
	double g2, rho, s;                           // g_min^2, rho, f 2^-l
};

// P at (x0 + fx, y0 + fy) (k = y0 wl + x0): along x, then y, each a + f (b - a)
template <typename T>
__device__ __forceinline__ double bilinear(const T *P, long long k, int wl, double fx, double fy)
{
	const double a = (double)P[k], b = (double)P[k + 1], c = (double)P[k + wl], d = (double)P[k + wl + 1];
	const double top = __dadd_rn(a, __dmul_rn(fx, __dsub_rn(b, a)));
	const double bot = __dadd_rn(c, __dmul_rn(fx, __dsub_rn(d, c)));
	return __dadd_rn(top, __dmul_rn(fy, __dsub_rn(bot, top)));
}

// pixel i's photometric Jacobian row J and residual r (zero, and false, when the pixel is skipped)
__device__ __forceinline__ bool photo_term(long long i, const Maps &S, const Maps &M, const Pose &T, const Step &st,
					   const Photo &ph, double *J)
{
	for (int k = 0; k < 7; k++) J[k] = 0.0;
	if (i >= (long long)st.hl * st.wl) return false;
	const double p0 = S.v[0][i];
	if (isnan(p0)) return false;                 // no source vertex
	double q[3];
	to_world(p0, S.v[1][i], S.v[2][i], T, q);
	if (!(q[2] > 0.0)) return false;
	const double xs = __dmul_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[0], q[2]), st.f), st.cx), st.scale);
	const double ys = __dmul_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[1], q[2]), st.f), st.cy), st.scale);
	const double u = floor(__dadd_rn(xs, 0.5)), v = floor(__dadd_rn(ys, 0.5));
	if (!(u >= 0.0 && u < st.wl && v >= 0.0 && v < st.hl)) return false;
	const long long j = (long long)v * st.wl + (long long)u;
	const double m0 = M.v[0][j];
	if (isnan(m0)) return false;                 // the reference view sees no surface there
	const double d[3] = {__dsub_rn(q[0], m0), __dsub_rn(q[1], M.v[1][j]), __dsub_rn(q[2], M.v[2][j])};
	const double dd = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
	if (!(dd <= st.d2)) return false;            // occluded in the reference view
	const double x0 = floor(xs), y0 = floor(ys);
	if (!(x0 >= 1.0 && __dadd_rn(x0, 1.0) <= st.wl - 2 && y0 >= 1.0 && __dadd_rn(y0, 1.0) <= st.hl - 2)) return false;
	const double fx = __dsub_rn(xs, x0), fy = __dsub_rn(ys, y0);
	const long long k = (long long)y0 * st.wl + (long long)x0;
	const double r = __dsub_rn(bilinear(ph.Ir, k, st.wl, fx, fy), (double)ph.Is[i]);
	const double gx = bilinear(ph.gx, k, st.wl, fx, fy), gy = bilinear(ph.gy, k, st.wl, fx, fy);
	if (!(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)) >= ph.g2 && fabs(r) <= ph.rho)) return false;
	const double a = __ddiv_rn(__dmul_rn(gx, ph.s), q[2]), b = __ddiv_rn(__dmul_rn(gy, ph.s), q[2]);
	const double c = __ddiv_rn(-__dadd_rn(__dmul_rn(a, q[0]), __dmul_rn(b, q[1])), q[2]);
	J[0] = __dsub_rn(__dmul_rn(q[1], c), __dmul_rn(q[2], b));
	J[1] = __dsub_rn(__dmul_rn(q[2], a), __dmul_rn(q[0], c));
	J[2] = __dsub_rn(__dmul_rn(q[0], b), __dmul_rn(q[1], a));
	J[3] = a;
	J[4] = b;
	J[5] = c;
	J[6] = r;
	return true;
}

// one block per chunk of 1024 pixels: the geometric terms (pixel_term) go through reduce_chunk into rows 0 .. 27 of
// part, and with PHOTO the photometric ones (photo_term) then through the same shared buffer into rows 28 .. 55;
// inliers[0] and [1] get the geometric and the photometric inlier counts
template <bool PHOTO>
__global__ void __launch_bounds__(RT) step_kernel(Maps S, Maps M, Pose T, Step st, Photo ph, double *__restrict__ part, int P,
						  unsigned long long *__restrict__ inliers)
{
	__shared__ double sh[NS * 128];
	const long long base = (long long)blockIdx.x * CH + threadIdx.x;
	int cg = 0, cp = 0;
	{
		double J[4][7];
#pragma unroll
		for (int p = 0; p < 4; p++) cg += pixel_term(base + p * RT, S, M, T, st, J[p]);
		reduce_chunk(J, sh, part, P);
	}
	if (PHOTO) {
		double J[4][7];
#pragma unroll
		for (int p = 0; p < 4; p++) cp += photo_term(base + p * RT, S, M, T, st, ph, J[p]);
		reduce_chunk(J, sh, part + (long long)NS * P, P);
	}
	const int tg = __reduce_add_sync(0xffffffffu, cg), tp = PHOTO ? __reduce_add_sync(0xffffffffu, cp) : 0;
	if ((threadIdx.x & 31) == 0) {
		if (tg) atomicAdd(inliers, (unsigned long long)tg);
		if (tp) atomicAdd(inliers + 1, (unsigned long long)tp);
	}
}

// `rows` rows of chunk sums (row k at part[k P]) padded with +0.0 from n to P (a power of two), reduced by stride halving
// in place; out = the rows' sums, then the geometric and the photometric inliers and the level's source vertices as int64
__global__ void __launch_bounds__(RED) chunk_reduce_kernel(double *__restrict__ part, int rows, int n, int P,
							   const unsigned long long *__restrict__ inliers,
							   const unsigned long long *__restrict__ nvert, double *__restrict__ out)
{
	for (long long e = threadIdx.x; e < (long long)rows * (P - n); e += RED) part[(e / (P - n)) * P + n + e % (P - n)] = 0.0;
	__syncthreads();
	for (int stride = P >> 1; stride >= 1; stride >>= 1) {
		for (long long e = threadIdx.x; e < (long long)rows * stride; e += RED) {
			const long long k = e / stride, i = e % stride;
			part[k * P + i] = __dadd_rn(part[k * P + i], part[k * P + i + stride]);
		}
		__syncthreads();
	}
	if (threadIdx.x < rows) out[threadIdx.x] = part[(long long)threadIdx.x * P];
	if (threadIdx.x == 0) {
		((long long *)out)[rows] = (long long)inliers[0];
		((long long *)out)[rows + 1] = (long long)inliers[1];
		((long long *)out)[rows + 2] = (long long)*nvert;
	}
}

bool camera_ok(float f, float cx, float cy) { return f > 0.f && isfinite(f) && isfinite(cx) && isfinite(cy); }

}  // namespace

struct mccnn_track {
	int H, W, device;
	int hl[LEVELS], wl[LEVELS];
	long long off[LEVELS];                        // each level's first double in a pyramid
	long long pyr;                                // doubles per pyramid
	int P;                                        // chunk sums per term: the level-0 chunk count rounded up to 2^k
	double *mem;                                  // source pyramid, model pyramid, 2 NS rows of P chunk sums, out
	unsigned long long *ctr;                      // geometric and photometric inliers, then the source vertices per level
	double *host;                                 // pinned: the up to 2 NS + 3 values read back per step
	float mf, mcx, mcy;                           // the model's camera
	bool have_source, have_model;
	// the photometric term's pyramids, allocated by the first mccnn_track_intensity
	long long ioff[LEVELS], npix;                 // each level's first pixel in an intensity pyramid; pixels per pyramid
	float *imem;                                  // the source's intensity pyramid, then the reference's
	double *pmem;                                 // the reference's g_x, g_y pyramids
	bool have_intensity[2];
};

namespace {

Maps level_maps(const mccnn_track *h, int which, int l)
{
	return maps_at(h->mem + which * h->pyr + h->off[l], (long long)h->hl[l] * h->wl[l]);
}

int build_pyramid(mccnn_track *h, int which, const float *src, const Cam &c, cudaStream_t s)
{
	if (which == 0) ADC_CUDA(cudaMemsetAsync(h->ctr + 2, 0, 8 * LEVELS, s));
	for (int l = 0; l < LEVELS; l++) {
		const long long np = (long long)h->hl[l] * h->wl[l];
		const Maps m = level_maps(h, which, l);
		vertex_kernel<<<adc_div_up(np, 256), 256, 0, s>>>(src, which, h->W, l, h->hl[l], h->wl[l], c, m,
								  which == 0 ? h->ctr + 2 + l : nullptr);
		normal_kernel<<<adc_div_up(np, 256), 256, 0, s>>>(h->hl[l], h->wl[l], m);
	}
	ADC_CHECK_LAUNCH();
	return 0;
}

int photo_alloc(mccnn_track *h)
{
	if (h->imem) return 0;
	long long at = 0;
	for (int l = 0; l < LEVELS; l++) {
		h->ioff[l] = at;
		at += (long long)h->hl[l] * h->wl[l];
	}
	h->npix = at;
	float *im = nullptr;
	double *pm = nullptr;
	cudaError_t e = cudaMalloc(&im, 4 * (size_t)(2 * at));
	if (e == cudaSuccess) e = cudaMalloc(&pm, 8 * (size_t)(2 * at));
	if (e != cudaSuccess) {
		if (im) cudaFree(im);
		return (int)e;
	}
	h->imem = im;
	h->pmem = pm;
	return 0;
}

}  // namespace

extern "C" {

int mccnn_track_create(mccnn_track **out, int H, int W, int device)
{
	if (!out) return ADCENSUS_EINVAL;
	*out = nullptr;
	if (H < 1 || W < 1) return ADCENSUS_EINVAL;
	if ((long long)H * W >= (1ll << 31)) return ADCENSUS_ELIMIT;
	int ndev = 0;
	ADC_CUDA(cudaGetDeviceCount(&ndev));
	if (device < 0 || device >= ndev) return ADCENSUS_EINVAL;
	DeviceScope dev(device);
	if (dev.rc) return dev.rc;
	mccnn_track *h = new mccnn_track();
	h->H = H;
	h->W = W;
	h->device = device;
	long long at = 0;
	for (int l = 0; l < LEVELS; l++) {
		h->hl[l] = (H + (1 << l) - 1) >> l;
		h->wl[l] = (W + (1 << l) - 1) >> l;
		h->off[l] = at;
		at += 6ll * h->hl[l] * h->wl[l];
	}
	h->pyr = at;
	const long long chunks = ((long long)H * W + CH - 1) / CH;
	h->P = 1;
	while (h->P < chunks) h->P <<= 1;
	const long long out_at = 2 * h->pyr + 2ll * NS * h->P;
	cudaError_t e = cudaMalloc(&h->mem, 8 * (size_t)(out_at + 2 * NS + 3) + 8 * (2 + LEVELS));
	if (e == cudaSuccess) e = cudaMallocHost(&h->host, 8 * (2 * NS + 3));
	if (e != cudaSuccess) {
		if (h->mem) cudaFree(h->mem);
		delete h;
		return (int)e;
	}
	h->ctr = (unsigned long long *)(h->mem + out_at + 2 * NS + 3);
	*out = h;
	return 0;
}

int mccnn_track_source(mccnn_track *h, const float *disp, float f, float cx, float cy, float fB, float doffs, float max_depth,
		       adcensus_stream_t stream)
{
	if (!h || !disp || !camera_ok(f, cx, cy) || !(fB > 0.f && isfinite(fB) && isfinite(doffs) && max_depth > 0.f))
		return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	const int rc = build_pyramid(h, 0, disp, Cam{f, cx, cy, fB, doffs, max_depth}, adc_stream(stream));
	if (!rc) h->have_source = true;
	return rc;
}

int mccnn_track_model(mccnn_track *h, const float *depth, float f, float cx, float cy, adcensus_stream_t stream)
{
	if (!h || !depth || !camera_ok(f, cx, cy)) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	const int rc = build_pyramid(h, 1, depth, Cam{f, cx, cy, 1.f, 0.f, INFINITY}, adc_stream(stream));
	if (!rc) {
		h->have_model = true;
		h->mf = f;
		h->mcx = cx;
		h->mcy = cy;
	}
	return rc;
}

int mccnn_track_step(mccnn_track *h, int level, const double *pose12, double delta, double cos_theta, const double *gates,
		     double *sums, long long *counts, adcensus_stream_t stream)
{
	if (!h || !sums || !counts || level < 0 || level >= LEVELS || !h->have_source || !h->have_model) return ADCENSUS_EINVAL;
	if (!(delta > 0.0 && isfinite(delta) && cos_theta >= -1.0 && cos_theta <= 1.0)) return ADCENSUS_EINVAL;
	if (gates && !(h->have_intensity[0] && h->have_intensity[1])) return ADCENSUS_EINVAL;
	if (gates && !(gates[0] >= 0.0 && isfinite(gates[0]) && gates[1] >= 0.0 && isfinite(gates[1]))) return ADCENSUS_EINVAL;
	Pose T;
	int rc = check_pose(pose12, &T);
	if (rc) return rc;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	const int hl = h->hl[level], wl = h->wl[level];
	const int n = (int)(((long long)hl * wl + CH - 1) / CH);
	int P = 1;
	while (P < n) P <<= 1;
	const int rows = gates ? 2 * NS : NS;
	double *part = h->mem + 2 * h->pyr, *out = part + 2ll * NS * h->P;
	const double scale = ldexp(1.0, -level);
	const Step st{hl, wl, (double)h->mf, (double)h->mcx, (double)h->mcy, scale, delta * delta, cos_theta};
	const Maps S = level_maps(h, 0, level), M = level_maps(h, 1, level);
	ADC_CUDA(cudaMemsetAsync(h->ctr, 0, 16, s));
	if (gates) {
		const long long o = h->ioff[level];
		const Photo ph{h->imem + o, h->imem + h->npix + o, h->pmem + o, h->pmem + h->npix + o, gates[0] * gates[0], gates[1],
			       (double)h->mf * scale};
		step_kernel<true><<<n, RT, 0, s>>>(S, M, T, st, ph, part, P, h->ctr);
	} else {
		step_kernel<false><<<n, RT, 0, s>>>(S, M, T, st, Photo{}, part, P, h->ctr);
	}
	chunk_reduce_kernel<<<1, RED, 0, s>>>(part, rows, n, P, h->ctr, h->ctr + 2 + level, out);
	ADC_CHECK_LAUNCH();
	ADC_CUDA(cudaMemcpyAsync(h->host, out, 8 * (rows + 3), cudaMemcpyDeviceToHost, s));
	ADC_CUDA(cudaStreamSynchronize(s));
	for (int k = 0; k < rows; k++) sums[k] = h->host[k];
	for (int k = 0; k < 3; k++) counts[k] = ((const long long *)h->host)[rows + k];
	return 0;
}

int mccnn_track_maps(const mccnn_track *h, int which, int level, double *vertices, double *normals, adcensus_stream_t stream)
{
	if (!h || !vertices || !normals || which < 0 || which > 1 || level < 0 || level >= LEVELS) return ADCENSUS_EINVAL;
	if (!(which ? h->have_model : h->have_source)) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	const size_t b = 24 * (size_t)h->hl[level] * h->wl[level];
	const double *p = h->mem + which * h->pyr + h->off[level];
	cudaStream_t s = adc_stream(stream);
	ADC_CUDA(cudaMemcpyAsync(vertices, p, b, cudaMemcpyDeviceToDevice, s));
	ADC_CUDA(cudaMemcpyAsync(normals, p + 3ll * h->hl[level] * h->wl[level], b, cudaMemcpyDeviceToDevice, s));
	return 0;
}

int mccnn_track_intensity(mccnn_track *h, int which, const unsigned char *img, int nch, adcensus_stream_t stream)
{
	if (!h || !img || which < 0 || which > 1 || (nch != 1 && nch != 3)) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	int rc = photo_alloc(h);
	if (rc) return rc;
	cudaStream_t s = adc_stream(stream);
	float *I = h->imem + which * h->npix;
	const long long np = (long long)h->H * h->W;
	grey_kernel<<<adc_div_up(np, 256), 256, 0, s>>>(img, nch, np, I);
	for (int l = 0; l + 1 < LEVELS; l++) {
		const long long n2 = (long long)h->hl[l + 1] * h->wl[l + 1];
		down_kernel<<<adc_div_up(n2, 256), 256, 0, s>>>(I + h->ioff[l], h->hl[l], h->wl[l], I + h->ioff[l + 1], h->hl[l + 1],
								 h->wl[l + 1]);
	}
	if (which == 1)
		for (int l = 0; l < LEVELS; l++) {
			const long long np_l = (long long)h->hl[l] * h->wl[l];
			gradient_kernel<<<adc_div_up(np_l, 256), 256, 0, s>>>(I + h->ioff[l], h->hl[l], h->wl[l], h->pmem + h->ioff[l],
									     h->pmem + h->npix + h->ioff[l]);
		}
	ADC_CHECK_LAUNCH();
	h->have_intensity[which] = true;
	return 0;
}

int mccnn_track_intensity_maps(const mccnn_track *h, int which, int level, float *I, double *gx, double *gy,
			       adcensus_stream_t stream)
{
	if (!h || !I || which < 0 || which > 1 || level < 0 || level >= LEVELS || !h->have_intensity[which]) return ADCENSUS_EINVAL;
	if (which == 1 ? (!gx || !gy) : (gx || gy)) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	const long long np = (long long)h->hl[level] * h->wl[level], o = h->ioff[level];
	cudaStream_t s = adc_stream(stream);
	ADC_CUDA(cudaMemcpyAsync(I, h->imem + which * h->npix + o, 4 * (size_t)np, cudaMemcpyDeviceToDevice, s));
	if (which == 1) {
		ADC_CUDA(cudaMemcpyAsync(gx, h->pmem + o, 8 * (size_t)np, cudaMemcpyDeviceToDevice, s));
		ADC_CUDA(cudaMemcpyAsync(gy, h->pmem + h->npix + o, 8 * (size_t)np, cudaMemcpyDeviceToDevice, s));
	}
	return 0;
}

void mccnn_track_destroy(mccnn_track *h)
{
	if (!h) return;
	{
		DeviceScope dev(h->device);
		if (!dev.rc) {
			if (h->mem) cudaFree(h->mem);
			if (h->host) cudaFreeHost(h->host);
			if (h->imem) cudaFree(h->imem);
			if (h->pmem) cudaFree(h->pmem);
		}
	}
	delete h;
}

}  // extern "C"
