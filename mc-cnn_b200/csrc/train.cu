// train.cu -- training of the fast architecture's matching-cost network (main.lua:602-890, arch 'fast'), for sm_90a.
//
// * train_sample_kernel: make_patch (main.lua:607-619) per output pixel.  OpenCV's warpAffine with INTER_CUBIC and a
//   constant 0 border, restated operation by operation: the float 2x3 matrix inverted in double, source coordinates on
//   AB_BITS = 10 fixed point rounded to the 1/32-pixel grid, the float cubic table (A = -0.75), interior taps summed row by
//   row, border taps summed one by one onto 0; then * contrast + brightness in fp32.  Bit-identical to oracle/train.py.
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
#include <math.h>
#include <stdlib.h>

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

__global__ void train_sample_kernel(const float *__restrict__ X0, const float *__restrict__ X1, int n_img, int H, int W,
				    const mccnn_warp *__restrict__ warps, const int *__restrict__ slot, int n, int ws,
				    float *__restrict__ out)
{
	const long id = (long)blockIdx.x * blockDim.x + threadIdx.x;
	const int np = ws * ws;
	if (id >= (long)n * np) return;
	const int p = (int)(id / np), y = (int)(id % np) / ws, x = (int)(id % np) % ws;
	const mccnn_warp w = warps[(slot ? (long)*slot * n : 0) + p];
	float *dst = out + id;
	if (w.image < 0 || w.image >= n_img) { *dst = adc_nan(); return; }
	const float *src = (w.view ? X1 : X0) + (long)w.image * H * W;

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

// layer k's gradient: block (ci, co) writes G's 9 weights of (co, ci) and, for ci == 0, the bias of co
__global__ void __launch_bounds__(WG_NT) wgrad_kernel(Layout L, int k, const float *__restrict__ X, const float *__restrict__ act,
						      const float *__restrict__ dz, float *__restrict__ G)
{
	__shared__ float red[10][WG_NT];
	const int ci = blockIdx.x, co = blockIdx.y, fm = L.fm, cin = k ? fm : 1;
	const int so = side(L, k), si = so + 2;
	float acc[10];
#pragma unroll
	for (int j = 0; j < 10; j++) acc[j] = 0.f;
	for (int n = threadIdx.x; n < L.N; n += WG_NT) {
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
	for (int s = WG_NT / 2; s > 0; s >>= 1) {
		if (threadIdx.x < s)
#pragma unroll
			for (int j = 0; j < 10; j++) red[j][threadIdx.x] += red[j][threadIdx.x + s];
		__syncthreads();
	}
	if (threadIdx.x < 9) G[L.woff[k] + ((long)co * cin + ci) * 9 + threadIdx.x] = red[threadIdx.x][0];
	if (threadIdx.x == 9 && ci == 0) G[L.boff[k] + co] = red[9][0];
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

}  // namespace

struct mccnn_trainer {
	Layout L;
	int device, bufsz, smem, chunk, loss_cap, n_img, H, W;
	long nparam;
	float margin, mom;
	int pow2;
	const float *X0, *X1;
	float *P, *V, *G, *X, *act, *dz, *norm, *nout, *join, *gjoin, *hinge, *gout, *loss, *neg_lr;
	float neg_lr_host;
	int *ctr;
	mccnn_warp *warps;
	cudaStream_t cap;
	cudaGraphExec_t full, body;
};

static int enqueue_step(mccnn_trainer *h, cudaStream_t s, bool sample)
{
	const Layout &L = h->L;
	const int ws = L.ws;
	if (sample) {
		const long tot = (long)L.N * ws * ws;
		train_sample_kernel<<<adc_div_up(tot, 128), 128, 0, s>>>(h->X0, h->X1, h->n_img, h->H, h->W, h->warps, h->ctr, L.N,
								       ws, h->X);
	}
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

static int capture(mccnn_trainer *h, bool sample, cudaGraphExec_t *exec)
{
	cudaGraph_t g = nullptr;
	ADC_CUDA(cudaStreamBeginCapture(h->cap, cudaStreamCaptureModeThreadLocal));
	const int rc = enqueue_step(h, h->cap, sample);
	const cudaError_t e = cudaStreamEndCapture(h->cap, &g);
	if (rc) { if (g) cudaGraphDestroy(g); return rc; }
	ADC_CUDA(e);
	const cudaError_t ei = cudaGraphInstantiate(exec, g, 0);
	cudaGraphDestroy(g);
	return (int)ei;
}

static float **train_buffer(mccnn_trainer *h, int what, long *count)
{
	const Layout &L = h->L;
	const long N = L.N, fm = L.fm;
	struct { float **p; long n; } t[] = {
		{&h->P, h->nparam}, {&h->V, h->nparam}, {&h->G, h->nparam}, {&h->X, N * L.ws * L.ws},
		{&h->act, L.aoff[L.l1 - 1] + N * fm}, {&h->norm, N}, {&h->nout, N * fm}, {&h->join, N / 2},
		{&h->gjoin, N / 2}, {&h->hinge, N / 4}, {&h->gout, N * fm}, {&h->dz, L.aoff[L.l1 - 1] + N * fm},
		{&h->loss, h->loss_cap},
	};
	if (what < 0 || what >= (int)(sizeof(t) / sizeof(t[0]))) return nullptr;
	*count = t[what].n;
	return t[what].p;
}

extern "C" int mccnn_train_sample(const float *X0, const float *X1, int n_img, int H, int W, const mccnn_warp *warps, int n,
				  int ws, float *out, adcensus_stream_t stream)
{
	if (!X0 || !X1 || !warps || !out || n_img < 1 || H < 1 || W < 1 || n < 1 || ws < 1) return ADCENSUS_EINVAL;
	if ((long)n * ws * ws >= (1l << 31) || H > 32767 || W > 32767) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	train_sample_kernel<<<adc_div_up((long)n * ws * ws, 128), 128, 0, s>>>(X0, X1, n_img, H, W, warps, nullptr, n, ws, out);
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
	if (h->cap) cudaStreamDestroy(h->cap);
	long n;
	for (int what = 0; what < MCCNN_TRAIN_NBUF; what++) cudaFree(*train_buffer(h, what, &n));
	cudaFree(h->neg_lr);
	cudaFree(h->ctr);
	cudaFree(h->warps);
	cudaSetDevice(prev);
	free(h);
	return 0;
}

extern "C" int mccnn_trainer_create(mccnn_trainer **out, int l1, int fm, int bs, float margin, int pow, float mom,
				    const float *X0, const float *X1, int n_img, int H, int W, int chunk, int loss_cap,
				    int device, adcensus_stream_t stream)
{
	if (!out || !X0 || !X1 || l1 < 1 || fm < 1 || bs < 2 || (bs % 2) || (pow != 1 && pow != 2) || n_img < 1 || H < 1 ||
	    W < 1 || chunk < 1 || loss_cap < 1)
		return ADCENSUS_EINVAL;
	if (l1 > LMAX || fm > 128 || H > 32767 || W > 32767) return ADCENSUS_ELIMIT;
	*out = nullptr;
	mccnn_trainer *h = (mccnn_trainer *)calloc(1, sizeof(mccnn_trainer));
	if (!h) return ADCENSUS_EINVAL;
	Layout &L = h->L;
	L.l1 = l1; L.fm = fm; L.ws = 1 + 2 * l1; L.N = 2 * bs;
	long off = 0, aoff = 0;
	for (int k = 0; k < l1; k++) {
		const int cin = k ? fm : 1, s = L.ws - 2 * (k + 1);
		L.woff[k] = off; off += (long)fm * cin * 9;
		L.boff[k] = off; off += fm;
		L.aoff[k] = aoff; aoff += (long)L.N * fm * s * s;
	}
	h->nparam = off;
	h->bufsz = L.ws * L.ws;
	for (int k = 1; k < l1; k++) h->bufsz = h->bufsz > fm * (L.ws - 2 * k) * (L.ws - 2 * k) ? h->bufsz
											   : fm * (L.ws - 2 * k) * (L.ws - 2 * k);
	h->smem = 2 * h->bufsz * (int)sizeof(float);
	h->device = device; h->chunk = chunk; h->loss_cap = loss_cap; h->n_img = n_img; h->H = H; h->W = W;
	h->margin = margin; h->mom = mom; h->pow2 = pow == 2; h->X0 = X0; h->X1 = X1;
	h->neg_lr_host = 0.f;
	int prev = 0;
	cudaGetDevice(&prev);
	int rc = (int)cudaSetDevice(device);
	int optin = 0;
	if (!rc) rc = (int)cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
	if (!rc && h->smem > optin) rc = ADCENSUS_ELIMIT;
	if (!rc) rc = (int)cudaFuncSetAttribute(tower_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem);
	if (!rc) rc = (int)cudaFuncSetAttribute(tower_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem);
	for (int what = 0; what < MCCNN_TRAIN_NBUF && !rc; what++) {
		long n;
		float **p = train_buffer(h, what, &n);
		rc = (int)cudaMalloc((void **)p, (size_t)n * sizeof(float));
		if (!rc) rc = (int)cudaMemsetAsync(*p, 0, (size_t)n * sizeof(float), adc_stream(stream));
	}
	if (!rc) rc = (int)cudaMalloc((void **)&h->neg_lr, sizeof(float));
	if (!rc) rc = (int)cudaMemsetAsync(h->neg_lr, 0, sizeof(float), adc_stream(stream));
	if (!rc) rc = (int)cudaMalloc((void **)&h->ctr, 2 * sizeof(int));
	if (!rc) rc = (int)cudaMemsetAsync(h->ctr, 0, 2 * sizeof(int), adc_stream(stream));
	if (!rc) rc = (int)cudaMalloc((void **)&h->warps, (size_t)chunk * L.N * sizeof(mccnn_warp));
	if (!rc) rc = (int)cudaMemsetAsync(h->warps, 0, (size_t)chunk * L.N * sizeof(mccnn_warp), adc_stream(stream));
	if (!rc) rc = (int)cudaStreamCreateWithFlags(&h->cap, cudaStreamNonBlocking);
	if (!rc) rc = capture(h, true, &h->full);
	if (!rc) rc = capture(h, false, &h->body);
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

extern "C" int mccnn_trainer_run(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr, adcensus_stream_t stream)
{
	if (!h || !warps || nsteps < 0) return ADCENSUS_EINVAL;
	if (nsteps > h->chunk) return ADCENSUS_ELIMIT;
	if (!nsteps) return 0;
	cudaStream_t s = adc_stream(stream);
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(h->device);
	int rc = set_lr(h, lr, s);
	if (!rc) rc = (int)cudaMemcpyAsync(h->warps, warps, (size_t)nsteps * h->L.N * sizeof(mccnn_warp), cudaMemcpyDefault, s);
	if (!rc) rc = (int)cudaMemsetAsync(h->ctr, 0, sizeof(int), s);
	for (int i = 0; i < nsteps && !rc; i++) rc = (int)cudaGraphLaunch(h->full, s);
	cudaSetDevice(prev);
	return rc;
}

extern "C" int mccnn_trainer_step_patches(mccnn_trainer *h, const float *patches, double lr, adcensus_stream_t stream)
{
	if (!h || !patches) return ADCENSUS_EINVAL;
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
	if (!h || !train_buffer(h, what, &n)) return -1;
	return n;
}

extern "C" int mccnn_trainer_get(mccnn_trainer *h, int what, float *dst, adcensus_stream_t stream)
{
	long n = 0;
	float **p = h ? train_buffer(h, what, &n) : nullptr;
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
	return h ? 5 + h->L.l1 : -1;
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
