// train.cu -- training of the fast architecture's matching-cost network (main.lua:602-890, arch 'fast'), for sm_90a.
//
// * train_sample_kernel: make_patch (main.lua:607-619) per output pixel.  OpenCV's warpAffine with INTER_CUBIC and a
//   constant 0 border, restated operation by operation: the float 2x3 matrix inverted in double, source coordinates on
//   AB_BITS = 10 fixed point rounded to the 1/32-pixel grid, the float cubic table (A = -0.75), interior taps summed row by
//   row, border taps summed one by one onto 0; then * contrast + brightness in fp32.  Bit-identical to oracle/train.py.
//   It reads a table of stereo pairs (mccnn_train_pair), each with its own H x W: KITTI's (n_img, 1, H, W) stacks become
//   one pair per image, Middlebury gives one pair per (image, light, exposure).
// * One training step (net_tr + Margin2 + the momentum update, main.lua:852-874) in fp32 on the CUDA cores, five kernels
//   plus one per layer, captured once into a CUDA graph:
//     tower_fwd_kernel   one block per patch, every layer's activations in shared memory (and kept in global memory);
//     head_kernel        one block per sample (4 patches): Normalize2, StereoJoin1, Margin2 and their backward passes,
//                        with the reference's Normalize and Margin2 expressions (adcensus.cu:1284-1453);
//     tower_bwd_kernel   one block per patch: the gradient through the convolutions and ReLUs, layer by layer;
//     wgrad_kernel       per layer, one block per (output, input) plane pair: the 3x3 weight (and bias) gradient summed
//                        over the batch, each thread's patches in order, then a fixed shared-memory tree;
//     update_kernel      v = v * mom; v = v + (-lr) * g; p = p + v, each operation rounded; the loss (the hinge terms
//                        summed in order / (bs / 2)) goes to the per-step loss buffer.
//   No floating-point atomics anywhere: a step is a pure function of its inputs, bit for bit.
// * Arch 'slow' (main.lua:663-677 + BCECriterion2): the same sampler, graph, chunked warp parameters and update_kernel;
//   the tower, the Linear layers and their backward passes are gemm_kernel launches (see below), then slow_head_kernel
//   and wgrad_reduce_kernel.  The fast kernels above are not shared with it.
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

constexpr int LMAX = 8;
constexpr int WG_NT = 256;           // wgrad_kernel threads (a power of two: the tree)

struct Layout {
	int l1, fm, ws, N;               // N = 2 bs patches
	long woff[LMAX], boff[LMAX];     // into the flat parameter vector: W (fm, cin, 3, 3), b (fm)
	long aoff[LMAX];                 // into act / dz: layer k's (N, fm, s_k, s_k), s_k = ws - 2 (k + 1)
};

__device__ __forceinline__ int side(const Layout &L, int k) { return L.ws - 2 * (k + 1); }

// OpenCV's interpolateCubic in fp32 (A = -0.75), each operation rounded as the host compiler does it
__device__ __forceinline__ void cubic_coeffs(float x, float c[4])
{
	const float A = -0.75f;
	const float t = __fadd_rn(x, 1.f);
	c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, t), -3.75f), t), -6.f), t), -3.f);
	c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, x), 2.25f), x), x), 1.f);
	const float u = __fsub_rn(1.f, x);
	c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, u), 2.25f), u), u), 1.f);
	c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c[0]), c[1]), c[2]);
}

__device__ __forceinline__ int sat_short(int v) { return min(32767, max(-32768, v)); }

// the source of each patch is pairs[w.image].x0 or .x1, with that pair's own H x W (and so its own constant-0 border)
__global__ void train_sample_kernel(const mccnn_train_pair *__restrict__ pairs, int n_pairs,
				    const mccnn_warp *__restrict__ warps, const int *__restrict__ slot, int n, int ws,
				    float *__restrict__ out)
{
	const long id = (long)blockIdx.x * blockDim.x + threadIdx.x;
	const int np = ws * ws;
	if (id >= (long)n * np) return;
	const int p = (int)(id / np), y = (int)(id % np) / ws, x = (int)(id % np) % ws;
	const mccnn_warp w = warps[(slot ? (long)*slot * n : 0) + p];
	float *dst = out + id;
	if (w.image < 0 || w.image >= n_pairs) { *dst = adc_nan(); return; }
	const mccnn_train_pair pr = pairs[w.image];
	const int H = pr.H, W = pr.W;
	const float *src = w.view ? pr.x1 : pr.x0;

	// warpAffine: invert the forward matrix in double
	double M0 = w.m[0], M1 = w.m[1], M2 = w.m[2], M3 = w.m[3], M4 = w.m[4], M5 = w.m[5];
	double D = __dsub_rn(__dmul_rn(M0, M4), __dmul_rn(M1, M3));
	D = D != 0 ? __ddiv_rn(1.0, D) : 0.0;
	const double A11 = __dmul_rn(M4, D), A22 = __dmul_rn(M0, D);
	M0 = A11; M1 = __dmul_rn(M1, -D);
	M3 = __dmul_rn(M3, -D); M4 = A22;
	const double b1 = __dsub_rn(__dmul_rn(-M0, M2), __dmul_rn(M1, M5));
	const double b2 = __dsub_rn(__dmul_rn(-M3, M2), __dmul_rn(M4, M5));

	// WarpAffineInvoker: AB_BITS = 10, round_delta = 1024 / 32 / 2
	const int X0i = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M1, (double)y), b1), 1024.0)) + 16;
	const int Y0i = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M4, (double)y), b2), 1024.0)) + 16;
	const int Xf = (X0i + __double2int_rn(__dmul_rn(__dmul_rn(M0, (double)x), 1024.0))) >> 5;
	const int Yf = (Y0i + __double2int_rn(__dmul_rn(__dmul_rn(M3, (double)x), 1024.0))) >> 5;
	const int sx = sat_short(Xf >> 5) - 1, sy = sat_short(Yf >> 5) - 1;
	float cx[4], cy[4];
	cubic_coeffs(__fmul_rn(0.03125f, (float)(Xf & 31)), cx);
	cubic_coeffs(__fmul_rn(0.03125f, (float)(Yf & 31)), cy);

	// remapBicubic, float source, BORDER_CONSTANT 0
	float sum = 0.f;
	if ((unsigned)sx < (unsigned)max(W - 3, 0) && (unsigned)sy < (unsigned)max(H - 3, 0)) {
		for (int i = 0; i < 4; i++) {
			const float *s = src + (long)(sy + i) * W + sx;
			float row = __fmul_rn(s[0], __fmul_rn(cy[i], cx[0]));
			row = __fadd_rn(row, __fmul_rn(s[1], __fmul_rn(cy[i], cx[1])));
			row = __fadd_rn(row, __fmul_rn(s[2], __fmul_rn(cy[i], cx[2])));
			row = __fadd_rn(row, __fmul_rn(s[3], __fmul_rn(cy[i], cx[3])));
			sum = i == 0 ? row : __fadd_rn(sum, row);
		}
	} else if (!(sx >= W || sx + 4 <= 0 || sy >= H || sy + 4 <= 0)) {
		for (int i = 0; i < 4; i++) {
			if (sy + i < 0 || sy + i >= H) continue;
			for (int j = 0; j < 4; j++)
				if (sx + j >= 0 && sx + j < W)
					sum = __fadd_rn(sum, __fmul_rn(src[(long)(sy + i) * W + sx + j], __fmul_rn(cy[i], cx[j])));
		}
	}
	*dst = __fadd_rn(__fmul_rn(sum, w.contrast), w.brightness);             // dst:mul(contrast):add(brightness)
}

// out[co][y][x] = b[co] + sum_{ci,ky,kx} w[co][ci][ky][kx] in[ci][y+ky][x+kx], over the whole block
__device__ void conv_valid(const float *__restrict__ in, float *__restrict__ out, float *__restrict__ gout,
			   const float *__restrict__ w, const float *__restrict__ b, int cin, int fm, int si, int relu)
{
	const int so = si - 2, plane = so * so;
	for (int o = threadIdx.x; o < fm * plane; o += blockDim.x) {
		const int co = o / plane, y = (o % plane) / so, x = (o % plane) % so;
		const float *wc = w + (long)co * cin * 9;
		float acc = 0.f;
		for (int ci = 0; ci < cin; ci++) {
			const float *a = in + (ci * si + y) * si + x;
			const float *k = wc + ci * 9;
#pragma unroll
			for (int ky = 0; ky < 3; ky++)
#pragma unroll
				for (int kx = 0; kx < 3; kx++) acc = fmaf(__ldg(k + ky * 3 + kx), a[ky * si + kx], acc);
		}
		acc += __ldg(b + co);
		if (relu) acc = fmaxf(acc, 0.f);
		out[o] = acc;
		gout[o] = acc;
	}
}

__global__ void tower_fwd_kernel(Layout L, const float *__restrict__ X, const float *__restrict__ P, float *__restrict__ act,
				 int bufsz)
{
	extern __shared__ float sm[];
	float *in = sm, *out = sm + bufsz;
	const int n = blockIdx.x, np = L.ws * L.ws;
	for (int i = threadIdx.x; i < np; i += blockDim.x) in[i] = X[(long)n * np + i];
	__syncthreads();
	for (int k = 0; k < L.l1; k++) {
		const int cin = k ? L.fm : 1, si = L.ws - 2 * k;
		const int so = si - 2;
		conv_valid(in, out, act + L.aoff[k] + (long)n * L.fm * so * so, P + L.woff[k], P + L.boff[k], cin, L.fm, si,
			   k < L.l1 - 1);
		__syncthreads();
		float *t = in; in = out; out = t;
	}
}

// Normalize2 + StereoJoin1 + Margin2 and back, for one sample (patches 4i .. 4i + 3); blockDim = 4 fm
__global__ void head_kernel(Layout L, const float *__restrict__ act, float margin, int pow2, float *__restrict__ norm,
			    float *__restrict__ nout, float *__restrict__ join, float *__restrict__ gjoin,
			    float *__restrict__ hinge, float *__restrict__ gout, float *__restrict__ dz)
{
	const int fm = L.fm, i = blockIdx.x, q = threadIdx.x / fm, c = threadIdx.x % fm;
	const int nsample = L.N / 4;
	const float *F = act + L.aoff[L.l1 - 1] + (long)4 * i * fm;               // (4, fm): the last layer's output
	const long base = (long)4 * i * fm;
	const int id = q * fm + c;
	if (c == 0) {                                                            // Normalize_get_norm_ (adcensus.cu:1284)
		float sum = 0.0;
		for (int d = 0; d < fm; d++) {
			float x = F[q * fm + d];
			sum += x * x;
		}
		norm[4 * i + q] = sum + 1e-5;
	}
	__syncthreads();
	const float nq = norm[4 * i + q];
	nout[base + id] = F[id] / sqrtf(nq);                                     // Normalize_forward_ (:1300)
	__syncthreads();
	if (c == 0 && (q & 1) == 0) {                                            // StereoJoin1: cmul, then sum over planes
		float s = 0.f;
		for (int d = 0; d < fm; d++) s = __fadd_rn(s, __fmul_rn(nout[base + q * fm + d], nout[base + (q + 1) * fm + d]));
		join[2 * i + q / 2] = s;
	}
	__syncthreads();
	if (threadIdx.x == 0) {                                                  // Margin2_ (:1379-1423), then :div(bs / 2)
		const float pos = join[2 * i], neg = join[2 * i + 1];
		const float f = neg - pos + margin;
		float h, g0, g1;
		if (!pow2) {
			h = fmaxf(0, neg - pos + margin);
			g0 = -1. * (f > 0);
			g1 = f > 0;
		} else {
			float d = fmaxf(0, neg - pos + margin);
			h = d * d * 0.5;
			g0 = -f * (f > 0);
			g1 = f * (f > 0);
		}
		hinge[i] = h;
		gjoin[2 * i] = g0 / (float)nsample;
		gjoin[2 * i + 1] = g1 / (float)nsample;
	}
	__syncthreads();
	const float gq = gjoin[2 * i + q / 2];                                  // StereoJoin1 backward: partner * gradOutput
	gout[base + id] = __fmul_rn(nout[base + (q ^ 1) * fm + c], gq);
	__syncthreads();
	{                                                                        // Normalize_backward_input_ (:1335-1357)
		const float *grad_output = gout + base;
		const float *input = F;
		float denom = powf(nq, 1.5);
		float deriv = (nq - input[id] * input[id]) / denom * grad_output[id];
		float sum = 0;
		for (int d = 0; d < fm; d++) {
			if (d != c) {
				int ind = q * fm + d;
				sum += input[ind] * grad_output[ind];
			}
		}
		dz[L.aoff[L.l1 - 1] + base + id] = deriv - sum * input[id] / denom;
	}
}

// dz of layer k -> dz of layer k - 1 through layer k's weights and layer k - 1's ReLU, one block per patch
__global__ void tower_bwd_kernel(Layout L, const float *__restrict__ P, const float *__restrict__ act, float *__restrict__ dz,
				 int bufsz)
{
	extern __shared__ float sm[];
	float *g = sm, *ga = sm + bufsz;
	const int n = blockIdx.x, fm = L.fm;
	{
		const int s = side(L, L.l1 - 1);
		const float *src = dz + L.aoff[L.l1 - 1] + (long)n * fm * s * s;
		for (int i = threadIdx.x; i < fm * s * s; i += blockDim.x) g[i] = src[i];
	}
	__syncthreads();
	for (int k = L.l1 - 1; k >= 1; k--) {
		const int so = side(L, k), si = so + 2, plane = si * si;
		const float *w = P + L.woff[k];
		const float *a = act + L.aoff[k - 1] + (long)n * fm * plane;
		float *dst = dz + L.aoff[k - 1] + (long)n * fm * plane;
		for (int o = threadIdx.x; o < fm * plane; o += blockDim.x) {
			const int ci = o / plane, y = (o % plane) / si, x = (o % plane) % si;
			float acc = 0.f;
			for (int co = 0; co < fm; co++) {
				const float *k9 = w + ((long)co * fm + ci) * 9;
				const float *gz = g + co * so * so;
#pragma unroll
				for (int ky = 0; ky < 3; ky++) {
					const int yy = y - ky;
					if (yy < 0 || yy >= so) continue;
#pragma unroll
					for (int kx = 0; kx < 3; kx++) {
						const int xx = x - kx;
						if (xx < 0 || xx >= so) continue;
						acc = fmaf(__ldg(k9 + ky * 3 + kx), gz[yy * so + xx], acc);
					}
				}
			}
			const float v = a[o] > 0.f ? acc : 0.f;                              // ReLU(true): the output > 0
			ga[o] = v;
			dst[o] = v;
		}
		__syncthreads();
		float *t = g; g = ga; ga = t;
	}
}

// layer k's gradient over the L.N patches of X / act / dz with NT threads: thread t sums patches t, t + NT, ... in order,
// then a shared-memory tree with strides NT / 2 .. 1; block (ci, co) writes G's 9 weights of (co, ci) and, for ci == 0, the
// bias of co
template <int NT>
__device__ __forceinline__ void wgrad_block(const Layout &L, int k, const float *__restrict__ X, const float *__restrict__ act,
					    const float *__restrict__ dz, float *__restrict__ G)
{
	__shared__ float red[10][NT];
	const int ci = blockIdx.x, co = blockIdx.y, fm = L.fm, cin = k ? fm : 1;
	const int so = side(L, k), si = so + 2;
	float acc[10];
#pragma unroll
	for (int j = 0; j < 10; j++) acc[j] = 0.f;
	for (int n = threadIdx.x; n < L.N; n += NT) {
		const float *gz = dz + L.aoff[k] + ((long)n * fm + co) * so * so;
		const float *a = k ? act + L.aoff[k - 1] + ((long)n * fm + ci) * si * si : X + (long)n * si * si;
		for (int y = 0; y < so; y++)
			for (int x = 0; x < so; x++) {
				const float gv = gz[y * so + x];
#pragma unroll
				for (int ky = 0; ky < 3; ky++)
#pragma unroll
					for (int kx = 0; kx < 3; kx++) acc[ky * 3 + kx] = fmaf(gv, a[(y + ky) * si + x + kx], acc[ky * 3 + kx]);
				acc[9] += gv;
			}
	}
#pragma unroll
	for (int j = 0; j < 10; j++) red[j][threadIdx.x] = acc[j];
	__syncthreads();
	for (int s = NT / 2; s > 0; s >>= 1) {
		if (threadIdx.x < s)
#pragma unroll
			for (int j = 0; j < 10; j++) red[j][threadIdx.x] += red[j][threadIdx.x + s];
		__syncthreads();
	}
	if constexpr (NT >= 10) {
		if (threadIdx.x < 9) G[L.woff[k] + ((long)co * cin + ci) * 9 + threadIdx.x] = red[threadIdx.x][0];
		if (threadIdx.x == 9 && ci == 0) G[L.boff[k] + co] = red[9][0];
	} else {
		for (int j = threadIdx.x; j < 10; j += NT) {
			if (j < 9) G[L.woff[k] + ((long)co * cin + ci) * 9 + j] = red[j][0];
			else if (ci == 0) G[L.boff[k] + co] = red[9][0];
		}
	}
}

__global__ void __launch_bounds__(WG_NT) wgrad_kernel(Layout L, int k, const float *__restrict__ X, const float *__restrict__ act,
						      const float *__restrict__ dz, float *__restrict__ G)
{
	wgrad_block<WG_NT>(L, k, X, act, dz, G);
}

// Data parallel over R = WG_NT / NT ranks, rank r holding the patches n = r, r + R, ... as its local patches 0, 1, ...:
// wgrad_kernel's thread t = r + R u sums exactly the patches r + R u, r + R u + 256, ..., which are this rank's local
// patches u, u + NT, ...; the tree levels 128 .. R of wgrad_kernel only ever add a thread of residue r to another of
// residue r, and in local numbering they are levels NT / 2 .. 1.  So this kernel on the rank's patches writes to G the
// value wgrad_kernel's red[][r] holds after level R, bit for bit; wgrad_ranks_kernel runs the levels R / 2 .. 1.
template <int NT>
__global__ void __launch_bounds__(NT) wgrad_residue_kernel(Layout L, int k, const float *__restrict__ X,
							   const float *__restrict__ act, const float *__restrict__ dz,
							   float *__restrict__ G)
{
	wgrad_block<NT>(L, k, X, act, dz, G);
}

// wgrad_kernel's tree levels R / 2 .. 1 over the ranks' partial sums part (R, n), rank-major, in place; G = the root
__global__ void wgrad_ranks_kernel(float *__restrict__ part, int R, long n, float *__restrict__ G)
{
	const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	for (int s = R / 2; s > 0; s >>= 1)
		for (int t = 0; t < s; t++) part[t * n + i] = __fadd_rn(part[t * n + i], part[(t + s) * n + i]);
	G[i] = part[i];
}

__global__ void update_kernel(float *__restrict__ P, float *__restrict__ V, const float *__restrict__ G, long n, float mom,
			      const float *__restrict__ neg_lr, const float *__restrict__ hinge, int nsample,
			      float *__restrict__ loss, int loss_cap, int *__restrict__ ctr)
{
	const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) {
		float v = __fmul_rn(V[i], mom);
		v = __fadd_rn(v, __fmul_rn(*neg_lr, G[i]));
		V[i] = v;
		P[i] = __fadd_rn(P[i], v);
	}
	if (i == 0) {                                                            // Margin2: self.tmp:mean()
		float s = 0.f;
		for (int j = 0; j < nsample; j++) s = __fadd_rn(s, hinge[j]);
		if (ctr[1] < loss_cap) loss[ctr[1]] = s / (float)nsample;
		ctr[0]++;
		ctr[1]++;
	}
}

// ---- arch 'slow' (main.lua:663-677): the tower with a ReLU after every layer, Reshape(bs, 2 fm), l2 x [Linear, ReLU],
// Linear(nh2, 1), Sigmoid, BCECriterion2.  Every convolution and Linear, forward and backward, is one tiled fp32 GEMM
// (gemm_kernel) whose operands are read through an implicit-im2col functor; each output is one thread's fmaf chain in
// ascending k, and the weight gradients of the tower are split over k into partial sums added in split order.
constexpr int L2MAX = 4;
constexpr int BM = 64, BN = 64, BK = 16, GT = 256;  // gemm_kernel: 64 x 64 tiles, 4 x 4 outputs per thread

template <class Op>
__global__ void __launch_bounds__(GT) gemm_kernel(Op op)
{
	__shared__ __align__(16) float As[BK][BM + 4], Bs[BK][BN + 4];
	const int t = threadIdx.x, tx = t % 16, ty = t / 16;
	const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
	const int k0 = blockIdx.z * op.kchunk, k1 = min(op.K, k0 + op.kchunk);
	float acc[4][4];
#pragma unroll
	for (int i = 0; i < 4; i++)
#pragma unroll
		for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
	for (int kb = k0; kb < k1; kb += BK) {
#pragma unroll
		for (int i = 0; i < BM * BK / GT; i++) {
			const int e = t + GT * i, m = e / BK, k = e % BK;
			As[k][m] = m0 + m < op.M && kb + k < k1 ? op.a(m0 + m, kb + k) : 0.f;
		}
#pragma unroll
		for (int i = 0; i < BN * BK / GT; i++) {
			const int e = t + GT * i, k = e / BN, n = e % BN;
			Bs[k][n] = n0 + n < op.N && kb + k < k1 ? op.b(kb + k, n0 + n) : 0.f;
		}
		__syncthreads();
#pragma unroll
		for (int k = 0; k < BK; k++) {
			const float4 a = *(const float4 *)&As[k][ty * 4], b = *(const float4 *)&Bs[k][tx * 4];
			const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
			for (int i = 0; i < 4; i++)
#pragma unroll
				for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
		}
		__syncthreads();
	}
#pragma unroll
	for (int i = 0; i < 4; i++)
#pragma unroll
		for (int j = 0; j < 4; j++) {
			const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
			if (m < op.M && n < op.N) op.store(m, n, acc[i][j], blockIdx.z);
		}
}

// layer forward: out[n][co][y][x] = ReLU(sum_{ci,ky,kx} W[co][ci][ky][kx] in[n][ci][y+ky][x+kx] + b[co]);
// rows co, columns (n, y, x), k = (ci, ky, kx)
struct ConvFwd {
	int M, N, K, kchunk, cin, si, so;
	const float *__restrict__ in, *__restrict__ w, *__restrict__ bias;
	float *__restrict__ out;
	__device__ float a(int m, int k) const { return __ldg(w + (long)m * K + k); }
	__device__ float b(int k, int c) const
	{
		const int P = so * so, n = c / P, p = c % P, ci = k / 9, tap = k % 9;
		return in[((long)n * cin + ci) * si * si + (p / so + tap / 3) * si + p % so + tap % 3];
	}
	__device__ void store(int m, int c, float acc, int) const
	{
		const int P = so * so, n = c / P, p = c % P;
		out[((long)n * M + m) * P + p] = fmaxf(acc + __ldg(bias + m), 0.f);
	}
};

// gradient through layer k's weights and layer k - 1's ReLU: rows ci, columns (n, y, x) of layer k's input, k = (co, ky, kx)
struct ConvBwdData {
	int M, N, K, kchunk, fm, si, so;
	const float *__restrict__ w, *__restrict__ dz, *__restrict__ act;
	float *__restrict__ dst;
	__device__ float a(int m, int k) const { return __ldg(w + ((long)(k / 9) * fm + m) * 9 + k % 9); }
	__device__ float b(int k, int c) const
	{
		const int Pi = si * si, n = c / Pi, p = c % Pi, co = k / 9, tap = k % 9;
		const int y = p / si - tap / 3, x = p % si - tap % 3;
		return y >= 0 && y < so && x >= 0 && x < so ? dz[((long)n * fm + co) * so * so + y * so + x] : 0.f;
	}
	__device__ void store(int m, int c, float acc, int) const
	{
		const int Pi = si * si;
		const long i = ((long)(c / Pi) * fm + m) * Pi + c % Pi;
		dst[i] = act[i] > 0.f ? acc : 0.f;
	}
};

// layer k's weight and bias gradient, split over k: rows co, columns (ci, ky, kx) and a last column of ones (the bias),
// k = (n, y, x); split z writes its partial sums to part (nsplit, M, N)
struct ConvWgrad {
	int M, N, K, kchunk, cin, si, so;
	const float *__restrict__ dz, *__restrict__ in;
	float *__restrict__ part;
	__device__ float a(int m, int k) const
	{
		const int P = so * so;
		return dz[((long)(k / P) * M + m) * P + k % P];
	}
	__device__ float b(int k, int c) const
	{
		if (c == N - 1) return 1.f;
		const int P = so * so, n = k / P, p = k % P, ci = c / 9, tap = c % 9;
		return in[((long)n * cin + ci) * si * si + (p / so + tap / 3) * si + p % so + tap % 3];
	}
	__device__ void store(int m, int c, float acc, int z) const { part[((long)z * M + m) * N + c] = acc; }
};

// ConvWgrad's splits z0 .. z1 - 1 alone, launched as splits 0 .. z1 - z0 - 1: k is shifted by kbase = z0 kchunk and
// op.part points at split z0, K ends where split z1 - 1 ends.  Each split is the same fmaf chain over the same k-range
// as in the whole launch, so it writes the same bits.
struct ConvWgradRange {
	int M, N, K, kchunk;
	ConvWgrad op;
	int kbase;
	__device__ float a(int m, int k) const { return op.a(m, k + kbase); }
	__device__ float b(int k, int c) const { return op.b(k + kbase, c); }
	__device__ void store(int m, int c, float acc, int z) const { op.store(m, c, acc, z); }
};

// Linear + ReLU: Y (bs, out) = ReLU(X (bs, in) W^T + b)
struct FcFwd {
	int M, N, K, kchunk;
	const float *__restrict__ x, *__restrict__ w, *__restrict__ bias;
	float *__restrict__ y;
	__device__ float a(int m, int k) const { return x[(long)m * K + k]; }
	__device__ float b(int k, int c) const { return __ldg(w + (long)c * K + k); }
	__device__ void store(int m, int c, float acc, int) const { y[(long)m * N + c] = fmaxf(acc + __ldg(bias + c), 0.f); }
};

// Linear's input gradient dZ (bs, out) W -> through the previous ReLU (mask = its output); the first Linear also writes
// the reshape's gradient (raw, no mask)
struct FcBwdData {
	int M, N, K, kchunk;
	const float *__restrict__ dz, *__restrict__ w, *__restrict__ mask;
	float *__restrict__ dst, *__restrict__ raw;
	__device__ float a(int m, int k) const { return dz[(long)m * K + k]; }
	__device__ float b(int k, int c) const { return __ldg(w + (long)k * N + c); }
	__device__ void store(int m, int c, float acc, int) const
	{
		const long i = (long)m * N + c;
		if (raw) raw[i] = acc;
		dst[i] = mask[i] > 0.f ? acc : 0.f;
	}
};

// Linear's weight and bias gradient: rows out, columns in and a last column of ones, k = the batch row
struct FcWgrad {
	int M, N, K, kchunk;
	const float *__restrict__ dz, *__restrict__ x;
	float *__restrict__ gw, *__restrict__ gb;
	__device__ float a(int m, int k) const { return dz[(long)k * M + m]; }
	__device__ float b(int k, int c) const { return c == N - 1 ? 1.f : x[(long)k * (N - 1) + c]; }
	__device__ void store(int m, int c, float acc, int) const
	{
		if (c == N - 1) gb[m] = acc;
		else gw[(long)m * (N - 1) + c] = acc;
	}
};

// Linear(nh2, 1) + Sigmoid + BCECriterion2 (targets 0, 1, 0, 1, ...: main.lua:848-849) and back to the last hidden
// Linear's pre-ReLU gradient, plus the last Linear's weight and bias gradient; one block
__global__ void slow_head_kernel(int bs, int nh2, const float *__restrict__ X, const float *__restrict__ w,
				 const float *__restrict__ b, float *__restrict__ z, float *__restrict__ sig,
				 float *__restrict__ gin, float *__restrict__ term, float *__restrict__ dzo,
				 float *__restrict__ dz, float *__restrict__ gw, float *__restrict__ gb, float *__restrict__ loss)
{
	const float eps = 1e-12f, n = (float)bs;
	const int lane = threadIdx.x % 32, warp = threadIdx.x / 32, nwarp = blockDim.x / 32;
	for (int r = warp; r < bs; r += nwarp) {
		float acc = 0.f;
		for (int k = lane; k < nh2; k += 32) acc = fmaf(X[(long)r * nh2 + k], w[k], acc);
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
		if (lane == 0) {
			const float zr = acc + b[0], y = 1.f / (1.f + expf(-zr)), t = (float)(r & 1);
			z[r] = zr;
			sig[r] = y;
			// updateOutput: term3 = (log(x + eps) * t + log(1 - x + eps) * (1 - t)) / n
			const float t1 = 1.f - t, t2 = __fmul_rn(logf(__fadd_rn(__fsub_rn(1.f, y), eps)), t1);
			term[r] = __fdiv_rn(__fadd_rn(__fmul_rn(logf(__fadd_rn(y, eps)), t), t2), n);
			// updateGradInput: -((t / (x + eps) - (1 - t) / (1 - x + eps)) / n)
			const float g1 = __fdiv_rn(t1, __fadd_rn(__fsub_rn(1.f, y), eps));
			const float g = -__fdiv_rn(__fsub_rn(__fdiv_rn(t, __fadd_rn(y, eps)), g1), n);
			gin[r] = g;
			dzo[r] = __fmul_rn(__fmul_rn(g, __fsub_rn(1.f, y)), y);          // Sigmoid backward
		}
	}
	__syncthreads();
	for (int k = threadIdx.x; k < nh2; k += blockDim.x) {
		float acc = 0.f;
		for (int r = 0; r < bs; r++) acc = fmaf(dzo[r], X[(long)r * nh2 + k], acc);
		gw[k] = acc;
	}
	for (long i = threadIdx.x; i < (long)bs * nh2; i += blockDim.x) {
		const int r = (int)(i / nh2), k = (int)(i % nh2);
		dz[i] = X[i] > 0.f ? __fmul_rn(dzo[r], w[k]) : 0.f;
	}
	if (threadIdx.x == 0) {
		float s = 0.f, l = 0.f;
		for (int r = 0; r < bs; r++) {
			s = __fadd_rn(s, dzo[r]);
			l = __fadd_rn(l, term[r]);
		}
		gb[0] = s;
		*loss = -l;                                                          // -term3:sum()
	}
}

struct SlowLayout {
	int l2, nh2, nsplit[LMAX], kchunk[LMAX];
	long fwoff[L2MAX + 1], fboff[L2MAX + 1];  // the Linear layers' W (out, in), b (out) in the parameter vector
	long poff[LMAX];                          // each tower layer's partial sums in the split-k workspace
};

// the tower's weight and bias gradients: the partial sums of the splits, added in split order
__global__ void wgrad_reduce_kernel(Layout L, SlowLayout S, const float *__restrict__ part, float *__restrict__ G)
{
	const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= L.boff[L.l1 - 1] + L.fm) return;
	int k = 0;
	while (i >= L.boff[k] + L.fm) k++;
	const int cin9 = (k ? L.fm : 1) * 9, N = cin9 + 1;
	const long co = i < L.boff[k] ? (i - L.woff[k]) / cin9 : i - L.boff[k];
	const int c = i < L.boff[k] ? (int)((i - L.woff[k]) % cin9) : cin9;
	const float *p = part + S.poff[k] + co * N + c;
	float s = p[0];
	for (int z = 1; z < S.nsplit[k]; z++) s = __fadd_rn(s, p[(long)z * L.fm * N]);
	G[i] = s;
}

template <class Op>
void launch_gemm(const Op &op, int nsplit, cudaStream_t s)
{
	gemm_kernel<Op><<<dim3(adc_div_up(op.N, BN), adc_div_up(op.M, BM), nsplit), GT, 0, s>>>(op);
}

// split each tower layer's weight-gradient GEMM (K = N s_k^2) so that it has about 256 blocks of at least 256 k each; the
// split depends on the shapes only, so the summation order (and the bits) do not depend on the device
void split_k(const Layout &L, SlowLayout &S)
{
	long poff = 0;
	for (int k = 0; k < L.l1; k++) {
		const int cin = k ? L.fm : 1, s = L.ws - 2 * (k + 1), K = L.N * s * s;
		const int tiles = adc_div_up(L.fm, BM) * adc_div_up(cin * 9 + 1, BN);
		const int want = std::max(1, std::min(adc_div_up(256, tiles), adc_div_up(K, 256)));
		S.kchunk[k] = adc_div_up(adc_div_up(K, want), BK) * BK;
		S.nsplit[k] = adc_div_up(K, S.kchunk[k]);
		S.poff[k] = poff; poff += (long)S.nsplit[k] * L.fm * (cin * 9 + 1);
	}
}

// A slow shard's share of the batch: rank r of R owns the patches [b0, b1) = [N r / R, N (r + 1) / R) and, in each tower
// layer k, the weight-gradient splits whose first k-index falls in them, [z0[k], z1[k]) (each split has one owner).  It
// runs the tower forward and backward on [b0, e): e >= b1 is the end of the last patch its splits read.
struct SlowPlan {
	int b0, b1, e, z0[LMAX], z1[LMAX];
};

SlowPlan slow_plan(const Layout &L, const SlowLayout &S, int rank, int world)
{
	SlowPlan p;
	p.b0 = (int)((long)L.N * rank / world);
	p.b1 = (int)((long)L.N * (rank + 1) / world);
	p.e = p.b1;
	for (int k = 0; k < L.l1; k++) {
		const long P = (long)(L.ws - 2 * (k + 1)) * (L.ws - 2 * (k + 1)), K = L.N * P, kc = S.kchunk[k];
		p.z0[k] = (int)((p.b0 * P + kc - 1) / kc);
		p.z1[k] = (int)std::min<long>(S.nsplit[k], (p.b1 * P + kc - 1) / kc);
		if (p.z1[k] > p.z0[k]) p.e = std::max(p.e, (int)((std::min(K, p.z1[k] * kc) + P - 1) / P));
	}
	return p;
}

}  // namespace

struct mccnn_trainer {
	Layout L;
	int device, bufsz, smem, chunk, loss_cap, n_pairs;
	long nparam;
	float margin, mom;
	int pow2;
	mccnn_train_pair *pairs;                 // device copy of the creator's table
	float *P, *V, *G, *X, *act, *dz, *norm, *nout, *join, *gjoin, *hinge, *gout, *loss, *neg_lr;
	float neg_lr_host;
	int *ctr;
	mccnn_warp *warps;
	cudaStream_t cap;
	cudaGraphExec_t full, body;
	// arch 'slow' only
	int slow;
	SlowLayout S;
	float *rows, *fc, *sig, *bce_grad, *rows_grad, *fc_dz, *term, *dzo, *part, *bce_loss;
	// a shard (rank of world > 0 ranks).  'fast': L covers the rank's patches n = rank + world j as local patches j, Lh the
	// whole batch's last layer for head_kernel; nh the head's patches (L.N on one GPU).  'slow': L is the whole batch's,
	// `plan` the rank's patches and splits.  nw: the warp records of one step.
	int nh, rank, world, nmax, nw;
	int shard_launches;                      // the kernel nodes of the three segments' graphs
	SlowPlan plan;
	long ntower;
	Layout Lh;
	float *hact, *hdz, *gact, *gpart;        // the batch's last layer and its head dz; the two gathered buffers
	cudaGraphExec_t seg[3];
};

// The slow step on patches [n0, n1) and, per tower layer k, the weight-gradient splits [z0[k], z1[k]): the whole batch
// and every split on one GPU; a shard's range and splits (slow_plan) otherwise.  Stage 0 is the tower forward, stage 1
// the Linear layers, BCE and the backward passes, stage 2 the reduction of the splits and the update.  A patch's tower,
// forward and backward, reads no other patch, and each output of ConvFwd / ConvBwdData is one thread's fmaf chain over
// k, so a patch gets the same bits in any column range.
static int enqueue_slow_stage(mccnn_trainer *h, cudaStream_t s, int stage, int n0, int n1, const int *z0, const int *z1)
{
	const Layout &L = h->L;
	const SlowLayout &S = h->S;
	const int bs = L.N / 2, fm = L.fm, nh2 = S.nh2, l2 = S.l2, n = n1 - n0;
	if (stage == 0) {
		for (int k = 0; k < L.l1; k++) {                                 // tower forward
			const int cin = k ? fm : 1, si = L.ws - 2 * k, so = si - 2;
			const ConvFwd op{fm, n * so * so, cin * 9, cin * 9, cin, si, so,
					 (k ? h->act + L.aoff[k - 1] : h->X) + (long)n0 * cin * si * si, h->P + L.woff[k],
					 h->P + L.boff[k], h->act + L.aoff[k] + (long)n0 * fm * so * so};
			launch_gemm(op, 1, s);
		}
	} else if (stage == 1) {
		const float *x = h->rows;
		for (int j = 0; j < l2; j++) {                                   // Linear + ReLU
			const int in = j ? nh2 : 2 * fm;
			const FcFwd op{bs, nh2, in, in, x, h->P + S.fwoff[j], h->P + S.fboff[j], h->fc + (long)j * bs * nh2};
			launch_gemm(op, 1, s);
			x = op.y;
		}
		slow_head_kernel<<<1, 512, 0, s>>>(bs, nh2, x, h->P + S.fwoff[l2], h->P + S.fboff[l2],
						  h->fc + (long)l2 * bs * nh2, h->sig, h->bce_grad, h->term, h->dzo,
						  h->fc_dz + (long)(l2 - 1) * bs * nh2, h->G + S.fwoff[l2], h->G + S.fboff[l2],
						  h->bce_loss);
		for (int j = l2 - 1; j >= 0; j--) {                              // Linear backward
			const int in = j ? nh2 : 2 * fm;
			const float *dz = h->fc_dz + (long)j * bs * nh2, *xj = j ? h->fc + (long)(j - 1) * bs * nh2 : h->rows;
			const FcBwdData op{bs, in, nh2, nh2, dz, h->P + S.fwoff[j], xj,
					   j ? h->fc_dz + (long)(j - 1) * bs * nh2 : h->dz + L.aoff[L.l1 - 1],
					   j ? nullptr : h->rows_grad};
			launch_gemm(op, 1, s);
			const FcWgrad og{nh2, in + 1, bs, bs, dz, xj, h->G + S.fwoff[j], h->G + S.fboff[j]};
			launch_gemm(og, 1, s);
		}
		for (int k = L.l1 - 1; k >= 1; k--) {                            // tower backward
			const int so = L.ws - 2 * (k + 1), si = so + 2;
			const long o = (long)n0 * fm * si * si;
			const ConvBwdData op{fm, n * si * si, fm * 9, fm * 9, fm, si, so, h->P + L.woff[k],
					     h->dz + L.aoff[k] + (long)n0 * fm * so * so, h->act + L.aoff[k - 1] + o,
					     h->dz + L.aoff[k - 1] + o};
			launch_gemm(op, 1, s);
		}
		for (int k = 0; k < L.l1; k++) {                                 // tower weight gradients, split over k
			const int cin = k ? fm : 1, so = L.ws - 2 * (k + 1);
			const ConvWgrad op{fm, cin * 9 + 1, L.N * so * so, S.kchunk[k], cin, so + 2, so, h->dz + L.aoff[k],
					   k ? h->act + L.aoff[k - 1] : h->X, h->part + S.poff[k]};
			if (z0[k] == 0 && z1[k] == S.nsplit[k]) {
				launch_gemm(op, S.nsplit[k], s);
			} else if (z1[k] > z0[k]) {
				const int kbase = z0[k] * S.kchunk[k];
				ConvWgradRange r{op.M, op.N, std::min(op.K, z1[k] * S.kchunk[k]) - kbase, op.kchunk, op, kbase};
				r.op.part += (long)z0[k] * op.M * op.N;
				launch_gemm(r, z1[k] - z0[k], s);
			}
		}
	} else {
		const long ntower = L.boff[L.l1 - 1] + fm;
		wgrad_reduce_kernel<<<adc_div_up(ntower, 256), 256, 0, s>>>(L, S, h->part, h->G);
		update_kernel<<<adc_div_up(h->nparam, 256), 256, 0, s>>>(h->P, h->V, h->G, h->nparam, h->mom, h->neg_lr,
									 h->bce_loss, 1, h->loss, h->loss_cap, h->ctr);
	}
	ADC_CHECK_LAUNCH();
	return 0;
}

static int enqueue_slow(mccnn_trainer *h, cudaStream_t s)
{
	int z0[LMAX] = {}, rc = 0;
	for (int stage = 0; stage < 3 && !rc; stage++) rc = enqueue_slow_stage(h, s, stage, 0, h->L.N, z0, h->S.nsplit);
	return rc;
}

static int enqueue_step(mccnn_trainer *h, cudaStream_t s, bool sample)
{
	const Layout &L = h->L;
	const int ws = L.ws;
	if (sample) {
		const long tot = (long)L.N * ws * ws;
		train_sample_kernel<<<adc_div_up(tot, 128), 128, 0, s>>>(h->pairs, h->n_pairs, h->warps, h->ctr, L.N, ws, h->X);
	}
	if (h->slow) return enqueue_slow(h, s);
	tower_fwd_kernel<<<L.N, 256, h->smem, s>>>(L, h->X, h->P, h->act, h->bufsz);
	head_kernel<<<L.N / 4, 4 * L.fm, 0, s>>>(L, h->act, h->margin, h->pow2, h->norm, h->nout, h->join, h->gjoin, h->hinge,
						  h->gout, h->dz);
	tower_bwd_kernel<<<L.N, 256, h->smem, s>>>(L, h->P, h->act, h->dz, h->bufsz);
	for (int k = 0; k < L.l1; k++)
		wgrad_kernel<<<dim3(k ? L.fm : 1, L.fm), WG_NT, 0, s>>>(L, k, h->X, h->act, h->dz, h->G);
	update_kernel<<<adc_div_up(h->nparam, 256), 256, 0, s>>>(h->P, h->V, h->G, h->nparam, h->mom, h->neg_lr, h->hinge,
								 L.N / 4, h->loss, h->loss_cap, h->ctr);
	ADC_CHECK_LAUNCH();
	return 0;
}

// the patches n = q, q + R, ... of N: rank q's share
static int shard_count(int N, int R, int q) { return (N - q + R - 1) / R; }

// wgrad_residue_kernel<WG_NT / R>, by log2(R)
using WgradFn = void (*)(Layout, int, const float *, const float *, const float *, float *);
static const WgradFn RESIDUE_KERNELS[] = {wgrad_residue_kernel<256>, wgrad_residue_kernel<128>, wgrad_residue_kernel<64>,
					  wgrad_residue_kernel<32>,  wgrad_residue_kernel<16>,  wgrad_residue_kernel<8>,
					  wgrad_residue_kernel<4>,   wgrad_residue_kernel<2>,   wgrad_residue_kernel<1>};
static_assert(WG_NT == 256, "one residue kernel per power of two up to WG_NT");

// One step of a shard, segment `seg` of three.  'slow': enqueue_slow_stage on the plan's patches and splits, the sampler
// first; the caller all-gathers the last layer's rows after segment 0 and the split partials after segment 1.  'fast':
// the caller all-gathers gact after segment 0 and gpart after segment 1 (every rank's slot from its owner):
//   0  the sampler and the tower on the rank's patches; its last layer -> gact slot `rank`
//   1  the batch's last layer from gact in batch order -> head_kernel on the whole batch (as on one GPU) -> the rank's
//      rows of its dz -> tower_bwd and wgrad_residue_kernel on the rank's patches -> gpart slot `rank`
//   2  wgrad_ranks_kernel: the gradient; update_kernel
static int enqueue_shard(mccnn_trainer *h, cudaStream_t s, int seg)
{
	const Layout &L = h->L;
	if (h->slow) {                          // the all-gathers: the tower's last layer (ROWS), then the split partials
		const SlowPlan &p = h->plan;
		if (seg == 0)
			train_sample_kernel<<<adc_div_up((long)h->nw * L.ws * L.ws, 128), 128, 0, s>>>(
				h->pairs, h->n_pairs, h->warps, h->ctr, h->nw, L.ws, h->X + (long)p.b0 * L.ws * L.ws);
		return enqueue_slow_stage(h, s, seg, p.b0, p.e, p.z0, p.z1);
	}
	const int fm = L.fm, R = h->world, r = h->rank, last = L.l1 - 1;
	const size_t row = (size_t)fm * sizeof(float);
	if (seg == 0) {
		const long tot = (long)L.N * L.ws * L.ws;
		train_sample_kernel<<<adc_div_up(tot, 128), 128, 0, s>>>(h->pairs, h->n_pairs, h->warps, h->ctr, L.N, L.ws, h->X);
		tower_fwd_kernel<<<L.N, 256, h->smem, s>>>(L, h->X, h->P, h->act, h->bufsz);
		ADC_CUDA(cudaMemcpyAsync(h->gact + (long)r * h->nmax * fm, h->act + L.aoff[last], L.N * row,
					 cudaMemcpyDeviceToDevice, s));
	} else if (seg == 1) {
		for (int q = 0; q < R; q++)                                      // rank q's patch j is patch q + R j
			ADC_CUDA(cudaMemcpy2DAsync(h->hact + (long)q * fm, R * row, h->gact + (long)q * h->nmax * fm, row, row,
						   shard_count(h->nh, R, q), cudaMemcpyDeviceToDevice, s));
		head_kernel<<<h->nh / 4, 4 * fm, 0, s>>>(h->Lh, h->hact, h->margin, h->pow2, h->norm, h->nout, h->join, h->gjoin,
							 h->hinge, h->gout, h->hdz);
		ADC_CUDA(cudaMemcpy2DAsync(h->dz + L.aoff[last], row, h->hdz + (long)r * fm, R * row, row, L.N,
					   cudaMemcpyDeviceToDevice, s));
		tower_bwd_kernel<<<L.N, 256, h->smem, s>>>(L, h->P, h->act, h->dz, h->bufsz);
		int lg = 0;
		while ((1 << lg) < R) lg++;
		for (int k = 0; k < L.l1; k++)
			RESIDUE_KERNELS[lg]<<<dim3(k ? fm : 1, fm), WG_NT / R, 0, s>>>(L, k, h->X, h->act, h->dz,
											 h->gpart + (long)r * h->ntower);
	} else {
		wgrad_ranks_kernel<<<adc_div_up(h->ntower, 256), 256, 0, s>>>(h->gpart, R, h->ntower, h->G);
		update_kernel<<<adc_div_up(h->nparam, 256), 256, 0, s>>>(h->P, h->V, h->G, h->nparam, h->mom, h->neg_lr, h->hinge,
									 h->nh / 4, h->loss, h->loss_cap, h->ctr);
	}
	ADC_CHECK_LAUNCH();
	return 0;
}

template <class Enqueue>
static int capture_with(mccnn_trainer *h, Enqueue enqueue, cudaGraphExec_t *exec, int *kernels = nullptr)
{
	cudaGraph_t g = nullptr;
	ADC_CUDA(cudaStreamBeginCapture(h->cap, cudaStreamCaptureModeThreadLocal));
	const int rc = enqueue(h->cap);
	const cudaError_t e = cudaStreamEndCapture(h->cap, &g);
	if (rc) { if (g) cudaGraphDestroy(g); return rc; }
	ADC_CUDA(e);
	if (kernels) {                                                           // add the graph's kernel launches
		size_t n = 0;
		cudaGraphGetNodes(g, nullptr, &n);
		std::vector<cudaGraphNode_t> nodes(n);
		cudaGraphGetNodes(g, nodes.data(), &n);
		for (cudaGraphNode_t v : nodes) {
			cudaGraphNodeType t;
			if (cudaGraphNodeGetType(v, &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) ++*kernels;
		}
	}
	const cudaError_t ei = cudaGraphInstantiate(exec, g, 0);
	cudaGraphDestroy(g);
	return (int)ei;
}

static int capture(mccnn_trainer *h, bool sample, cudaGraphExec_t *exec)
{
	return capture_with(h, [&](cudaStream_t s) { return enqueue_step(h, s, sample); }, exec);
}

// the trainer's buffers by id: the public MCCNN_TRAIN_* ids, then the slow step's internal ones (id >= MCCNN_TRAIN_NBUF).
// nullptr for an id that does not apply to the handle's arch.
enum { TRAIN_FC_DZ = MCCNN_TRAIN_NBUF, TRAIN_TERM, TRAIN_DZO, TRAIN_PART, TRAIN_BCE_LOSS, TRAIN_NALL };

static float **train_buffer(mccnn_trainer *h, int what, long *count)
{
	const Layout &L = h->L;
	const SlowLayout &S = h->S;
	const long N = L.N, fm = L.fm, bs = N / 2, nh2 = S.nh2, Nh = h->nh;
	const int F = !h->slow, Sl = h->slow;
	struct { float **p; long n; int ok; } t[] = {
		{&h->P, h->nparam, 1}, {&h->V, h->nparam, 1}, {&h->G, h->nparam, 1}, {&h->X, N * L.ws * L.ws, 1},
		{&h->act, L.aoff[L.l1 - 1] + N * fm, 1}, {&h->norm, Nh, F}, {&h->nout, Nh * fm, F}, {&h->join, Nh / 2, F},
		{&h->gjoin, Nh / 2, F}, {&h->hinge, Nh / 4, F}, {&h->gout, Nh * fm, F}, {&h->dz, L.aoff[L.l1 - 1] + N * fm, 1},
		{&h->loss, h->loss_cap, 1},
		{&h->rows, bs * 2 * fm, Sl}, {&h->fc, S.l2 * bs * nh2 + bs, Sl}, {&h->sig, bs, Sl}, {&h->bce_grad, bs, Sl},
		{&h->rows_grad, bs * 2 * fm, Sl},
		{&h->fc_dz, S.l2 * bs * nh2, Sl}, {&h->term, bs, Sl}, {&h->dzo, bs, Sl},
		{&h->part, Sl ? S.poff[L.l1 - 1] + (long)S.nsplit[L.l1 - 1] * fm * (fm * 9 + 1) : 0, Sl}, {&h->bce_loss, 1, Sl},
	};
	static_assert(sizeof(t) / sizeof(t[0]) == TRAIN_NALL, "one entry per buffer id");
	if (what < 0 || what >= TRAIN_NALL || !t[what].ok) return nullptr;
	*count = t[what].n;
	return t[what].p;
}

// ROWS is a view of the tower's last layer (N, fm, 1, 1) = (bs, 2 fm), not an allocation of its own
static bool owned(int what) { return what != MCCNN_TRAIN_ROWS; }

static int check_pairs(const mccnn_train_pair *pairs, int n_pairs)
{
	if (!pairs || n_pairs < 1) return ADCENSUS_EINVAL;
	for (int i = 0; i < n_pairs; i++) {
		const mccnn_train_pair &p = pairs[i];
		if (!p.x0 || !p.x1 || p.H < 1 || p.W < 1) return ADCENSUS_EINVAL;
		if (p.H > 32767 || p.W > 32767) return ADCENSUS_ELIMIT;
	}
	return 0;
}

extern "C" int mccnn_train_sample_pairs(const mccnn_train_pair *pairs, int n_pairs, const mccnn_warp *warps, int n, int ws,
					float *out, adcensus_stream_t stream)
{
	if (!pairs || n_pairs < 1 || !warps || !out || n < 1 || ws < 1) return ADCENSUS_EINVAL;
	if ((long)n * ws * ws >= (1l << 31)) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	std::vector<mccnn_train_pair> t(n_pairs);
	ADC_CUDA(cudaMemcpyAsync(t.data(), pairs, t.size() * sizeof(mccnn_train_pair), cudaMemcpyDeviceToHost, s));
	ADC_CUDA(cudaStreamSynchronize(s));
	const int rc = check_pairs(t.data(), n_pairs);
	if (rc) return rc;
	train_sample_kernel<<<adc_div_up((long)n * ws * ws, 128), 128, 0, s>>>(pairs, n_pairs, warps, nullptr, n, ws, out);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int mccnn_trainer_destroy(mccnn_trainer *h)
{
	if (!h) return 0;
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	if (h->full) cudaGraphExecDestroy(h->full);
	if (h->body) cudaGraphExecDestroy(h->body);
	for (cudaGraphExec_t g : h->seg)
		if (g) cudaGraphExecDestroy(g);
	if (h->cap) cudaStreamDestroy(h->cap);
	long n;
	for (int what = 0; what < TRAIN_NALL; what++) {
		float **p = train_buffer(h, what, &n);
		if (p && owned(what)) cudaFree(*p);
	}
	cudaFree(h->neg_lr);
	cudaFree(h->ctr);
	cudaFree(h->warps);
	cudaFree(h->pairs);
	for (float *p : {h->hact, h->hdz, h->gact, h->gpart}) cudaFree(p);
	cudaSetDevice(prev);
	free(h);
	return 0;
}

// the limits of include/adcensus_b200.h's mccnn_trainer_create, in the order EINVAL, the pair table, ELIMIT
static int check_config(mccnn_trainer **out, const mccnn_trainer_config *c, const mccnn_train_pair *pairs, int n_pairs)
{
	if (!out || !c || (c->slow != 0 && c->slow != 1) || c->l1 < 1 || c->fm < 1 || c->bs < 2 || (c->bs % 2) ||
	    c->chunk < 1 || c->loss_cap < 1 || (c->slow ? c->l2 < 1 || c->nh2 < 1 : c->pow != 1 && c->pow != 2) ||
	    c->world < 1 || (c->world & (c->world - 1)) || c->rank < 0 || c->rank >= c->world)
		return ADCENSUS_EINVAL;
	const int rc = check_pairs(pairs, n_pairs);
	if (rc) return rc;
	if (c->l1 > LMAX || c->fm > 128 || c->world > WG_NT || c->world > 2l * c->bs ||
	    (c->slow && (c->fm % 16 || c->l2 > L2MAX || (c->nh2 != 128 && c->nh2 != 256 && c->nh2 != 384) ||
			 2l * c->bs * c->fm * (1 + 2 * c->l1) * (1 + 2 * c->l1) >= (1l << 31))))
		return ADCENSUS_ELIMIT;
	return 0;
}

extern "C" int mccnn_trainer_create(mccnn_trainer **out, const mccnn_trainer_config *cfg, const mccnn_train_pair *pairs,
				    int n_pairs, int device, adcensus_stream_t stream)
{
	if (out) *out = nullptr;
	const int bad = check_config(out, cfg, pairs, n_pairs);
	if (bad) return bad;
	// a one-GPU trainer has world 0: run / step_patches and the shard_* calls tell it from a shard by that
	const int slow = cfg->slow, l1 = cfg->l1, fm = cfg->fm, l2 = cfg->l2, nh2 = cfg->nh2, bs = cfg->bs,
		  chunk = cfg->chunk, rank = cfg->rank, world = cfg->world > 1 ? cfg->world : 0;
	mccnn_trainer *h = (mccnn_trainer *)calloc(1, sizeof(mccnn_trainer));
	if (!h) return ADCENSUS_EINVAL;
	h->slow = slow;
	Layout &L = h->L;
	L.l1 = l1; L.fm = fm; L.ws = 1 + 2 * l1; L.N = world && !slow ? shard_count(2 * bs, world, rank) : 2 * bs;
	h->nh = 2 * bs; h->rank = rank; h->world = world;
	long off = 0, aoff = 0;
	for (int k = 0; k < l1; k++) {
		const int cin = k ? fm : 1, s = L.ws - 2 * (k + 1);
		L.woff[k] = off; off += (long)fm * cin * 9;
		L.boff[k] = off; off += fm;
		L.aoff[k] = aoff; aoff += (long)L.N * fm * s * s;
	}
	if (slow) {
		SlowLayout &S = h->S;
		S.l2 = l2; S.nh2 = nh2;
		for (int j = 0; j <= l2; j++) {
			const int in = j ? nh2 : 2 * fm, o = j < l2 ? nh2 : 1;
			S.fwoff[j] = off; off += (long)o * in;
			S.fboff[j] = off; off += o;
		}
		split_k(L, S);
		if (world) h->plan = slow_plan(L, S, rank, world);
	}
	h->nparam = off;
	h->bufsz = L.ws * L.ws;
	for (int k = 1; k < l1; k++) h->bufsz = h->bufsz > fm * (L.ws - 2 * k) * (L.ws - 2 * k) ? h->bufsz
											   : fm * (L.ws - 2 * k) * (L.ws - 2 * k);
	h->smem = 2 * h->bufsz * (int)sizeof(float);
	h->device = device; h->chunk = chunk; h->loss_cap = cfg->loss_cap; h->n_pairs = n_pairs;
	h->margin = cfg->margin; h->mom = cfg->mom; h->pow2 = cfg->pow == 2;
	h->neg_lr_host = 0.f;
	int prev = 0;
	cudaGetDevice(&prev);
	int rc = (int)cudaSetDevice(device);
	if (!slow) {
		if (!rc) rc = adc_smem_optin(tower_fwd_kernel, h->smem);
		if (!rc) rc = adc_smem_optin(tower_bwd_kernel, h->smem);
	}
	for (int what = 0; what < TRAIN_NALL && !rc; what++) {
		long n;
		float **p = train_buffer(h, what, &n);
		if (!p || !owned(what)) continue;
		rc = (int)cudaMalloc((void **)p, (size_t)n * sizeof(float));
		if (!rc) rc = (int)cudaMemsetAsync(*p, 0, (size_t)n * sizeof(float), adc_stream(stream));
	}
	if (slow) h->rows = h->act + L.aoff[l1 - 1];
	if (!rc) rc = (int)cudaMalloc((void **)&h->neg_lr, sizeof(float));
	if (!rc) rc = (int)cudaMemsetAsync(h->neg_lr, 0, sizeof(float), adc_stream(stream));
	if (!rc) rc = (int)cudaMalloc((void **)&h->ctr, 2 * sizeof(int));
	if (!rc) rc = (int)cudaMemsetAsync(h->ctr, 0, 2 * sizeof(int), adc_stream(stream));
	h->nw = slow && world ? h->plan.e - h->plan.b0 : L.N;
	if (!rc) rc = (int)cudaMalloc((void **)&h->warps, (size_t)chunk * h->nw * sizeof(mccnn_warp));
	if (!rc) rc = (int)cudaMemsetAsync(h->warps, 0, (size_t)chunk * h->nw * sizeof(mccnn_warp), adc_stream(stream));
	if (!rc) rc = (int)cudaMalloc((void **)&h->pairs, (size_t)n_pairs * sizeof(mccnn_train_pair));
	if (!rc) rc = (int)cudaMemcpy(h->pairs, pairs, (size_t)n_pairs * sizeof(mccnn_train_pair), cudaMemcpyHostToDevice);
	if (world && !slow) {
		h->Lh = L;
		h->Lh.N = h->nh;
		h->Lh.aoff[l1 - 1] = 0;
		h->nmax = shard_count(h->nh, world, 0);
		h->ntower = L.boff[l1 - 1] + fm;
		const long n[4] = {(long)h->nh * fm, (long)h->nh * fm, (long)world * h->nmax * fm, world * h->ntower};
		float **p[4] = {&h->hact, &h->hdz, &h->gact, &h->gpart};
		for (int i = 0; i < 4 && !rc; i++) {
			rc = (int)cudaMalloc((void **)p[i], (size_t)n[i] * sizeof(float));
			if (!rc) rc = (int)cudaMemsetAsync(*p[i], 0, (size_t)n[i] * sizeof(float), adc_stream(stream));
		}
	}
	if (!rc) rc = (int)cudaStreamCreateWithFlags(&h->cap, cudaStreamNonBlocking);
	if (world) {
		for (int seg = 0; seg < 3 && !rc; seg++)
			rc = capture_with(h, [&](cudaStream_t s) { return enqueue_shard(h, s, seg); }, &h->seg[seg],
					  &h->shard_launches);
	} else {
		if (!rc) rc = capture(h, true, &h->full);
		if (!rc) rc = capture(h, false, &h->body);
	}
	if (!rc) rc = (int)cudaStreamSynchronize(adc_stream(stream));
	cudaSetDevice(prev);
	if (rc) {
		mccnn_trainer_destroy(h);
		return rc;
	}
	*out = h;
	return 0;
}

static int set_lr(mccnn_trainer *h, double lr, cudaStream_t s)
{
	const float v = (float)(-lr);                                           // add(-opt.lr, grads[i]): the scalar as float
	if (v == h->neg_lr_host && v != 0.f) return 0;
	h->neg_lr_host = v;
	ADC_CUDA(cudaMemcpyAsync(h->neg_lr, &h->neg_lr_host, sizeof(float), cudaMemcpyHostToDevice, s));
	return 0;
}

// the start of a chunk of nsteps steps: the lr, the steps' nw warp records each, the step counter back to 0
static int begin_chunk(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr, cudaStream_t s)
{
	int rc = set_lr(h, lr, s);
	if (!rc) rc = (int)cudaMemcpyAsync(h->warps, warps, (size_t)nsteps * h->nw * sizeof(mccnn_warp), cudaMemcpyDefault, s);
	if (!rc) rc = (int)cudaMemsetAsync(h->ctr, 0, sizeof(int), s);
	return rc;
}

extern "C" int mccnn_trainer_run(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr, adcensus_stream_t stream)
{
	if (!h || h->world || !warps || nsteps < 0) return ADCENSUS_EINVAL;
	if (nsteps > h->chunk) return ADCENSUS_ELIMIT;
	if (!nsteps) return 0;
	cudaStream_t s = adc_stream(stream);
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	int rc = begin_chunk(h, warps, nsteps, lr, s);
	for (int i = 0; i < nsteps && !rc; i++) rc = (int)cudaGraphLaunch(h->full, s);
	cudaSetDevice(prev);
	return rc;
}

extern "C" int mccnn_trainer_shard_begin(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr,
					 adcensus_stream_t stream)
{
	if (!h || !h->world || !warps || nsteps < 0) return ADCENSUS_EINVAL;
	if (nsteps > h->chunk) return ADCENSUS_ELIMIT;
	if (!nsteps) return 0;
	cudaStream_t s = adc_stream(stream);
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	const int rc = begin_chunk(h, warps, nsteps, lr, s);
	cudaSetDevice(prev);
	return rc;
}

extern "C" int mccnn_trainer_shard_segment(mccnn_trainer *h, int segment, adcensus_stream_t stream)
{
	if (!h || !h->world || segment < 0 || segment > 2) return ADCENSUS_EINVAL;
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	const int rc = (int)cudaGraphLaunch(h->seg[segment], adc_stream(stream));
	cudaSetDevice(prev);
	return rc;
}

extern "C" int mccnn_trainer_shard_buffer(mccnn_trainer *h, int what, float **ptr, long long *count)
{
	if (!h || !h->world || !ptr || !count || (what != MCCNN_SHARD_TOWER_OUT && what != MCCNN_SHARD_WGRAD_PART))
		return ADCENSUS_EINVAL;
	const Layout &L = h->L;
	const bool tower = what == MCCNN_SHARD_TOWER_OUT;
	long n = 0;
	if (h->slow) {
		*ptr = tower ? h->act + L.aoff[L.l1 - 1] : h->part;
		train_buffer(h, tower ? MCCNN_TRAIN_ROWS : TRAIN_PART, &n);
	} else {
		*ptr = tower ? h->gact : h->gpart;
		n = h->world * (tower ? (long)h->nmax * L.fm : h->ntower);
	}
	*count = n;
	return 0;
}

extern "C" int mccnn_trainer_shard_pieces(mccnn_trainer *h, int what)
{
	if (!h || !h->world || (what != MCCNN_SHARD_TOWER_OUT && what != MCCNN_SHARD_WGRAD_PART)) return ADCENSUS_EINVAL;
	return h->slow && what == MCCNN_SHARD_WGRAD_PART ? h->L.l1 : 1;
}

extern "C" int mccnn_trainer_shard_slot(mccnn_trainer *h, int what, int piece, int rank, long long *offset,
					long long *count)
{
	if (!h || !h->world || !offset || !count || rank < 0 || rank >= h->world || piece < 0 ||
	    piece >= mccnn_trainer_shard_pieces(h, what))
		return ADCENSUS_EINVAL;
	const Layout &L = h->L;
	if (h->slow) {
		const SlowPlan p = slow_plan(L, h->S, rank, h->world);
		if (what == MCCNN_SHARD_TOWER_OUT) {
			*offset = (long long)p.b0 * L.fm;
			*count = (long long)(p.b1 - p.b0) * L.fm;
		} else {
			const long per = (long)L.fm * ((piece ? L.fm : 1) * 9 + 1);        // one split's partial sums
			*offset = h->S.poff[piece] + p.z0[piece] * per;
			*count = std::max(0, p.z1[piece] - p.z0[piece]) * per;
		}
	} else {
		const long slot = what == MCCNN_SHARD_TOWER_OUT ? (long)h->nmax * L.fm : h->ntower;
		*offset = rank * slot;
		*count = slot;
	}
	return 0;
}

extern "C" int mccnn_trainer_slow_shard_plan(int l1, int fm, int bs, int rank, int world, long long *plan)
{
	if (l1 < 1 || l1 > LMAX || fm < 1 || bs < 1 || world < 1 || world > 2 * bs || rank < 0 || rank >= world || !plan)
		return ADCENSUS_EINVAL;
	Layout L{};
	L.l1 = l1; L.fm = fm; L.ws = 1 + 2 * l1; L.N = 2 * bs;
	SlowLayout S{};
	split_k(L, S);
	const SlowPlan p = slow_plan(L, S, rank, world);
	plan[0] = p.b0; plan[1] = p.b1; plan[2] = p.e;
	for (int k = 0; k < l1; k++) {
		plan[3 + 3 * k] = p.z0[k];
		plan[4 + 3 * k] = p.z1[k];
		plan[5 + 3 * k] = S.nsplit[k];
	}
	return 0;
}

extern "C" int mccnn_trainer_step_patches(mccnn_trainer *h, const float *patches, double lr, adcensus_stream_t stream)
{
	if (!h || h->world || !patches) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	int rc = set_lr(h, lr, s);
	if (!rc)
		rc = (int)cudaMemcpyAsync(h->X, patches, (size_t)h->L.N * h->L.ws * h->L.ws * sizeof(float), cudaMemcpyDefault, s);
	if (!rc) rc = (int)cudaGraphLaunch(h->body, s);
	cudaSetDevice(prev);
	return rc;
}

extern "C" long long mccnn_trainer_size(mccnn_trainer *h, int what)
{
	long n = 0;
	if (!h || what >= MCCNN_TRAIN_NBUF || !train_buffer(h, what, &n)) return -1;
	return n;
}

extern "C" int mccnn_trainer_get(mccnn_trainer *h, int what, float *dst, adcensus_stream_t stream)
{
	long n = 0;
	float **p = h && what < MCCNN_TRAIN_NBUF ? train_buffer(h, what, &n) : nullptr;
	if (!p || !dst) return ADCENSUS_EINVAL;
	return (int)cudaMemcpyAsync(dst, *p, (size_t)n * sizeof(float), cudaMemcpyDefault, adc_stream(stream));
}

extern "C" int mccnn_trainer_set(mccnn_trainer *h, int what, const float *src, adcensus_stream_t stream)
{
	long n = 0;
	float **p = h ? train_buffer(h, what, &n) : nullptr;
	if (!p || !src || (what != MCCNN_TRAIN_PARAMS && what != MCCNN_TRAIN_MOMENTA)) return ADCENSUS_EINVAL;
	return (int)cudaMemcpyAsync(*p, src, (size_t)n * sizeof(float), cudaMemcpyDefault, adc_stream(stream));
}

extern "C" int mccnn_trainer_reset_losses(mccnn_trainer *h, adcensus_stream_t stream)
{
	if (!h) return ADCENSUS_EINVAL;
	return (int)cudaMemsetAsync(h->ctr + 1, 0, sizeof(int), adc_stream(stream));
}

extern "C" int mccnn_trainer_launches_per_step(mccnn_trainer *h)
{
	if (!h) return -1;
	if (h->world) return h->shard_launches;
	return h->slow ? 3 + 3 * h->L.l1 + 3 * h->S.l2 : 5 + h->L.l1;
}

extern "C" int mccnn_randperm_swaps(long long *perm, long long n, long long i0, const unsigned *draws, long long k)
{
	if (!perm || !draws || i0 < 0 || k < 0 || i0 + k > (n > 0 ? n - 1 : 0)) return ADCENSUS_EINVAL;
	for (long long j = 0; j < k; j++) {
		const long long i = i0 + j, z = (long long)(draws[j] % (unsigned long long)(n - i));
		const long long t = perm[i];
		perm[i] = perm[i + z];
		perm[i + z] = t;
	}
	return 0;
}

extern "C" int mccnn_mb_sample_starts(const unsigned *raw, long long n_raw, int base, double d_exp, long long *starts,
				      long long cap, long long *count, long long *used)
{
	if ((!raw && n_raw) || n_raw < 0 || base < 0 || cap < 0 || (!starts && cap) || !count || !used) return ADCENSUS_EINVAL;
	long long pos = 0, k = 0;
	while (k < cap && pos + base + 4 <= n_raw) {
		const int extra = raw[pos + base + 2] * (1.0 / 4294967296.0) < d_exp;     // torch.uniform() < opt.d_exp
		if (pos + base + 4 + extra > n_raw) break;
		starts[k++] = pos;
		pos += base + 4 + extra;
	}
	*count = k;
	*used = pos;
	return 0;
}
