// scorer_head.cu -- the accurate ('slow') architecture's scorer head as ONE fused tensor-core kernel.
//
// Reference (main.lua:958-984, 688-695; SpatialConvolution1_fw.lua:11-31): for every disparity d the tower outputs are
// sliced (l = left[:, :, d:], r = right[:, :, :W-d]), stacked along channels (2 fm) and pushed through net_te2 =
// l2 x [per-pixel W x + b (cuBLAS addmm), ReLU], then W5 x + b5 (nh2 -> 1) and a sigmoid: 228 x 5 GEMM launches plus 228
// slice / concat copies per direction, activations through HBM between them.  The (H, W-d) result is the matching cost of
// disparity d, stored at vol[d, :, d:] (direction -1) and vol[d, :, :W-d] (direction +1): the same numbers, so they are
// computed ONCE here and written to both volumes.
//
// H100 design.  A tile is 64 consecutive pixels of one image row at one disparity = 64 rows of the per-pixel MLP; the
// whole chain runs on it without leaving the SM:
//   * wgmma (m64nNk16, bf16 operands, fp32 accumulation in registers) issued by two consumer warpgroups that split the
//     columns: warpgroup g computes the 64 x N/2 block of columns g N/2 .. (g + 1) N/2 (96 accumulator registers per
//     thread at nh2 = 384, so both fit next to the operand builders without spilling);
//   * fp32 parity through a bf16 SPLIT: x = hi + lo (two bf16), x . w ~= hi.whi + lo.whi + hi.wlo -- three MMAs per K step
//     into the same accumulator (the dropped lo.wlo term is 2^-16 relative): ~1e-6 relative per layer, the north star's
//     1e-4 holds with two orders of margin.  nterms = 1 (plain bf16, ~1e-3) is selectable for speed;
//   * activations stay on chip: the A operand of a layer (64 x K, hi and lo, 96 KB at K = 384) lives in shared memory in
//     the canonical K-major no-swizzle core-matrix layout [K/8][64 rows][16 bytes]; once both warpgroups have finished the
//     layer's MMAs, the epilogue (+ bias, ReLU, split, straight from the accumulator fragment) writes the next layer's
//     A operand in place;
//   * weights stream: pre-split once into per-K-step slabs [2 chunks][N][8 bf16] (exactly the shared-memory image the MMA
//     wants), fetched by ONE thread with cp.async.bulk into a ring (full / empty mbarriers; each warpgroup frees a slot once
//     its MMAs on it have completed); they are L2-resident (2.1 MB for kitti) and shared by all CTAs;
//   * layer 1 takes its rows straight from the (fm, H, W) tower outputs (left pixel x, right pixel x - d: coalesced loads
//     along x), the last hidden layer's epilogue folds the nh2 -> 1 product, bias and sigmoid and stores the two volumes.
// A CTA owns (image row, 64-pixel tile) and loops over the disparities.  Roles: warps 0-7 (two warpgroups) build the tile,
// issue the MMAs and run the epilogues, warp 8 streams weights.
//
// Roofline: tensor-bound.  Per valid (pixel, d): 2 * (2 fm * nh2 + (l2 - 1) * nh2^2) flop = 1.06 MFLOP for kitti
// (fm 112, nh2 384, l2 4), x 3 for the split.
#include <stdlib.h>
#include <string.h>

#include "wgmma.cuh"

namespace {

constexpr int SH_M = 64;                     // rows per tile (wgmma M)
constexpr int SH_ACHUNK = SH_M * 16;         // one 8-wide K chunk of an A operand: [64 rows][8 bf16]
constexpr int SH_NMAX = 384, SH_KMAX = 384, SH_LMAX = 4;
constexpr int SH_SLAB = 2 * SH_NMAX * 16;    // ring slot: one K = 16 step of B, [2 chunks][N][8 bf16]
constexpr int SH_ABYTES = (SH_KMAX / 8) * SH_ACHUNK;
constexpr int SH_NCONS = 256;                // two consumer warpgroups
constexpr int SH_NT = SH_NCONS + 32;         // + weight producer warp

template <int NTERMS>
struct SHCfg {
	static constexpr int NSLOT = NTERMS == 3 ? 8 : 12;
	static constexpr int OFF_AHI = 0;
	static constexpr int OFF_ALO = SH_ABYTES;
	static constexpr int OFF_RING = NTERMS == 3 ? 2 * SH_ABYTES : SH_ABYTES;
	static constexpr int OFF_CONST = OFF_RING + NSLOT * SH_SLAB;            // floats: bias[LMAX][NMAX], w5[NMAX], b5
	static constexpr int NCONST = SH_LMAX * SH_NMAX + SH_NMAX + 4;
	static constexpr int OFF_BAR = OFF_CONST + NCONST * 4;                   // full[NSLOT], empty[NSLOT]
	static constexpr int OFF_PART = OFF_BAR + 2 * NSLOT * 8;                 // [64] partial dot products of warpgroup 1
	static constexpr int SMEM = OFF_PART + SH_M * 4;
	static_assert(SMEM <= 232448, "shared memory budget");
};

struct SHParams {
	const float *featL, *featR;
	float *volL, *volR;
	const unsigned char *wslabs;     // per layer, per K step: [hi slab][lo slab], slab = [2][N][8] bf16
	const float *consts;             // bias of the hidden layers [L][NMAX], w5[NMAX], b5
	long slab_off[SH_LMAX];          // byte offset of layer l's first slab
	int nk[SH_LMAX];                 // K steps (of 16) of layer l
	int fm, N, L, H, W, D;
};

// NH = N / 2: the columns of one warpgroup
template <int NTERMS, int NH>
__global__ void __launch_bounds__(SH_NT, 1)
scorer_head_kernel(const SHParams p)
{
	using C = SHCfg<NTERMS>;
	constexpr int NSLOT = C::NSLOT;
	extern __shared__ __align__(128) unsigned char sh_smem[];
	unsigned char *a_hi = sh_smem + C::OFF_AHI, *a_lo = sh_smem + C::OFF_ALO;
	unsigned char *ring = sh_smem + C::OFF_RING;
	float *cst = reinterpret_cast<float *>(sh_smem + C::OFF_CONST);
	uint64_t *bar_full = reinterpret_cast<uint64_t *>(sh_smem + C::OFF_BAR);
	uint64_t *bar_empty = bar_full + NSLOT;
	float *part = reinterpret_cast<float *>(sh_smem + C::OFF_PART);

	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int x0 = blockIdx.x * SH_M, y = blockIdx.y;
	const int N = p.N, L = p.L, W = p.W;
	const long HW = (long)p.H * W;
	// disparities with at least one valid pixel in this tile: d <= x (adcensus / main.lua:967-968), d < D
	const int xl = min(x0 + SH_M, W) - 1;
	const int nd = min(p.D, xl + 1);
	const uint32_t slab_bytes = (uint32_t)N * 32u;

	if (tid == 0) {
		for (int s = 0; s < NSLOT; s++) {
			mbar_init(&bar_full[s], 1);
			mbar_init(&bar_empty[s], 2);           // one arrival per consumer warpgroup
		}
		mbar_fence_init();
	}
	for (int i = tid; i < C::NCONST; i += SH_NT) cst[i] = p.consts[i];
	__syncthreads();

	if (warp == 8) {
		// ------------------------------------------------------------ weight producer
		if (lane == 0) {
			unsigned it = 0;
			for (int t = 0; t < nd; t++)
				for (int l = 0; l < L; l++) {
					const unsigned char *src = p.wslabs + p.slab_off[l];
					for (int ks = 0; ks < p.nk[l]; ks++)
						for (int part = 0; part < (NTERMS == 3 ? 2 : 1); part++, it++) {
							const int s = it % NSLOT;
							if (it >= (unsigned)NSLOT) sh_wait(&bar_empty[s], ((it / NSLOT) - 1) & 1);
							mbar_arrive_expect_tx(&bar_full[s], slab_bytes);
							sh_bulk_load(ring + s * SH_SLAB, src + ((long)ks * 2 + part) * slab_bytes, slab_bytes, &bar_full[s]);
						}
				}
		}
		return;
	}
	// ---------------------------------------------------------------- consumers: two warpgroups
	const int g = tid >> 7, t = tid & 127;
	const int n0 = g * NH;                                   // first column of this warpgroup
	const int r0 = 16 * (t >> 5) + (lane >> 2), q = lane & 3; // accumulator rows r0, r0 + 8; columns 8 j + 2 q (+1)
	const int fm = p.fm, nc1 = 2 * fm / 8, ncl = fm / 8;
	const uint32_t a_hi_s = tma_smem_addr(a_hi), a_lo_s = tma_smem_addr(a_lo), ring_s = tma_smem_addr(ring);
	const uint32_t lbo_b = (uint32_t)N * 16u;
	const float *w5 = cst + SH_LMAX * SH_NMAX;
	const float b5 = w5[SH_NMAX];
	// layer-1 builder: row m, K chunks m4, m4 + 4, ... (four threads per row, loads coalesced along x)
	const int m = tid & 63, m4 = tid >> 6;
	const int xb = x0 + m;
	float acc[NH / 2];
#pragma unroll
	for (int i = 0; i < NH / 2; i++) acc[i] = 0.0f;
	unsigned it = 0;
	for (int d = 0; d < nd; d++) {
		// layer 1 input: [left pixel x ; right pixel x - d], main.lua:967-970, two K chunks (16 loads) in flight
		{
			const bool rowok = xb < W && xb >= d;
			const float *pl = p.featL + (long)y * W + (rowok ? xb : 0);
			const float *pr = p.featR + (long)y * W + (rowok ? xb - d : 0);
			for (int kc0 = m4; kc0 < nc1; kc0 += 8) {
				float v[2][8];
#pragma unroll
				for (int u = 0; u < 2; u++) {
					const int kc = kc0 + 4 * u;
					const float *src = kc < ncl ? pl + (long)(8 * kc) * HW : pr + (long)(8 * (kc - ncl)) * HW;
#pragma unroll
					for (int e = 0; e < 8; e++) v[u][e] = (rowok && kc < nc1) ? __ldg(src + (long)e * HW) : 0.0f;
				}
#pragma unroll
				for (int u = 0; u < 2; u++)
					if (kc0 + 4 * u < nc1) sh_store8<NTERMS>(a_hi, a_lo, SH_ACHUNK, kc0 + 4 * u, m, v[u]);
			}
		}
		fence_proxy_async_smem();              // generic stores -> visible to the tensor core's (async proxy) reads
		sh_bar(1, SH_NCONS);
		for (int l = 0; l < L; l++) {
			// ---- MMAs: one commit group per ring slot; a slot is freed once the group after it has been issued and
			// the one reading it has completed
			wg_fence_acc(acc);
			wg_fence();
			int pend = -1;
			for (int ks = 0; ks < p.nk[l]; ks++) {
				const uint64_t da_hi = sh_desc(a_hi_s + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
				const uint64_t da_lo = sh_desc(a_lo_s + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
#pragma unroll
				for (int part = 0; part < (NTERMS == 3 ? 2 : 1); part++, it++) {
					const int s = it % NSLOT;
					sh_wait_mma(&bar_full[s], (it / NSLOT) & 1);
					const uint64_t db = sh_desc(ring_s + s * SH_SLAB + n0 * 16, lbo_b, 128);
					if (part == 0) {              // w_hi slab: a_hi . w_hi (+ a_lo . w_hi)
						wg_mma<NH>(acc, da_hi, db, ks > 0);
						if (NTERMS == 3) wg_mma<NH>(acc, da_lo, db, 1);
					} else {                      // w_lo slab: a_hi . w_lo
						wg_mma<NH>(acc, da_hi, db, 1);
					}
					wg_commit();
					wg_wait<1>();
					sh_arrive_if(&bar_empty[pend < 0 ? 0 : pend], pend >= 0 && t == 0);
					pend = s;
				}
			}
			wg_wait<0>();
			wg_fence_acc(acc);
			sh_arrive_if(&bar_empty[pend], t == 0);
			sh_bar(1, SH_NCONS);                  // both warpgroups are done reading this layer's A operand
			const float *bias = cst + l * SH_NMAX;
			if (l + 1 < L) {
				// hidden layer: + bias, ReLU (SpatialConvolution1_fw.lua:21-27, cudnn.ReLU), next layer's operand in place
#pragma unroll
				for (int j = 0; j < NH / 8; j++) {
					const int c = n0 + 8 * j + 2 * q;
					const float bc = bias[c], bd = bias[c + 1];
					sh_store2<NTERMS>(a_hi, a_lo, SH_ACHUNK, c, r0, fmaxf(acc[4 * j] + bc, 0.0f), fmaxf(acc[4 * j + 1] + bd, 0.0f));
					sh_store2<NTERMS>(a_hi, a_lo, SH_ACHUNK, c, r0 + 8, fmaxf(acc[4 * j + 2] + bc, 0.0f), fmaxf(acc[4 * j + 3] + bd, 0.0f));
				}
				fence_proxy_async_smem();
				sh_bar(1, SH_NCONS);
			} else {
				// last hidden layer folded with the nh2 -> 1 layer and the sigmoid (main.lua:693-694)
				float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
				for (int j = 0; j < NH / 8; j++) {
					const int c = n0 + 8 * j + 2 * q;
					s0 = fmaf(fmaxf(acc[4 * j] + bias[c], 0.0f), w5[c], s0);
					s0 = fmaf(fmaxf(acc[4 * j + 1] + bias[c + 1], 0.0f), w5[c + 1], s0);
					s1 = fmaf(fmaxf(acc[4 * j + 2] + bias[c], 0.0f), w5[c], s1);
					s1 = fmaf(fmaxf(acc[4 * j + 3] + bias[c + 1], 0.0f), w5[c + 1], s1);
				}
				s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
				s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
				s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
				s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
				if (g == 1 && q == 0) {
					part[r0] = s0;
					part[r0 + 8] = s1;
				}
				sh_bar(1, SH_NCONS);
				if (g == 0 && q < 2) {
					const int r = r0 + 8 * q;
					const int x = x0 + r;
					const float z = ((q ? s1 : s0) + part[r]) + b5;
					const float sg = 1.0f / (1.0f + expf(-z));
					if (x < W && x >= d) {
						const long o = ((long)d * p.H + y) * W;
						if (p.volL) p.volL[o + x] = sg;           // main.lua:976, direction -1: columns d ..
						if (p.volR) p.volR[o + x - d] = sg;       //                direction +1: columns .. W - d
					}
				}
				sh_bar(1, SH_NCONS);                  // part[] and the A operand are free for the next disparity
			}
		}
	}
}

// weights (N x K fp32, row-major) -> slabs: per K step [hi: [2][N][8] bf16][lo: [2][N][8] bf16]
__global__ void sh_prep_kernel(const float *__restrict__ w, unsigned short *__restrict__ slabs, int N, int K)
{
	const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (long)N * K) return;
	const int n = (int)(i / K), k = (int)(i % K);
	const float v = w[i];
	const unsigned hb = __float_as_uint(v);
	// round to nearest even bf16 (finite weights)
	const unsigned hi = (hb + 0x7fffu + ((hb >> 16) & 1u)) >> 16;
	const float r = v - __uint_as_float(hi << 16);
	const unsigned rb = __float_as_uint(r);
	const unsigned lo = (rb + 0x7fffu + ((rb >> 16) & 1u)) >> 16;
	const int ks = k / 16, j = (k / 8) & 1, e = k & 7;
	const long slab = (long)N * 16;                       // bf16 elements per slab
	const long base = (long)ks * 2 * slab + ((long)j * N + n) * 8 + e;
	slabs[base] = (unsigned short)hi;
	slabs[base + slab] = (unsigned short)lo;
}

}  // namespace

struct mccnn_scorer_head {
	int fm, nh2, l2, device;
	unsigned char *wslabs;
	float *consts;
	long slab_off[SH_LMAX];
	int nk[SH_LMAX];
};

// W[i] (out_i x in_i, row-major) / b[i] (out_i) for i = 0 .. l2 (the last one is the nh2 -> 1 layer): DEVICE pointers,
// the layout of net_te2's SpatialConvolution1_fw modules (main.lua:688-695).
extern "C" int mccnn_scorer_head_create(mccnn_scorer_head **out, int fm, int nh2, int l2, const float *const *W, const float *const *b,
					 int device, adcensus_stream_t stream)
{
	if (!out || !W || !b || fm < 8 || nh2 < 128 || l2 < 1) return ADCENSUS_EINVAL;
	if (l2 > SH_LMAX || nh2 > SH_NMAX || (nh2 % 128) || (fm % 8) || 2 * fm > SH_KMAX) return ADCENSUS_ELIMIT;
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(device);
	cudaStream_t s = adc_stream(stream);
	mccnn_scorer_head *h = (mccnn_scorer_head *)calloc(1, sizeof(*h));
	if (!h) return ADCENSUS_EINVAL;
	h->fm = fm; h->nh2 = nh2; h->l2 = l2; h->device = device;
	int rc = 0;
	long total = 0;
	for (int l = 0; l < l2; l++) {
		const int K = l == 0 ? 2 * fm : nh2;
		h->nk[l] = (K + 15) / 16;
		h->slab_off[l] = total;
		total += (long)h->nk[l] * 2 * nh2 * 32;
	}
	rc = (int)cudaMalloc((void **)&h->wslabs, total);
	if (!rc) rc = (int)cudaMemsetAsync(h->wslabs, 0, total, s);            // K padding of layer 1 (2 fm not a multiple of 16)
	if (!rc) rc = (int)cudaMalloc((void **)&h->consts, SHCfg<3>::NCONST * sizeof(float));
	if (!rc) rc = (int)cudaMemsetAsync(h->consts, 0, SHCfg<3>::NCONST * sizeof(float), s);
	for (int l = 0; l < l2 && !rc; l++) {
		const int K = l == 0 ? 2 * fm : nh2;
		const long n = (long)nh2 * K;
		sh_prep_kernel<<<adc_div_up(n, 256), 256, 0, s>>>(W[l], (unsigned short *)(h->wslabs + h->slab_off[l]), nh2, K);
		rc = (int)cudaPeekAtLastError();
		if (!rc) rc = (int)cudaMemcpyAsync(h->consts + l * SH_NMAX, b[l], nh2 * sizeof(float), cudaMemcpyDeviceToDevice, s);
	}
	if (!rc) rc = (int)cudaMemcpyAsync(h->consts + SH_LMAX * SH_NMAX, W[l2], nh2 * sizeof(float), cudaMemcpyDeviceToDevice, s);
	if (!rc) rc = (int)cudaMemcpyAsync(h->consts + SH_LMAX * SH_NMAX + SH_NMAX, b[l2], sizeof(float), cudaMemcpyDeviceToDevice, s);
	if (!rc) rc = (int)cudaStreamSynchronize(s);
	cudaSetDevice(prev);
	if (rc) {
		cudaFree(h->wslabs);
		cudaFree(h->consts);
		free(h);
		return rc;
	}
	*out = h;
	return 0;
}

extern "C" void mccnn_scorer_head_destroy(mccnn_scorer_head *h)
{
	if (!h) return;
	cudaFree(h->wslabs);
	cudaFree(h->consts);
	free(h);
}

template <int NH>
static int sh_launch(const SHParams &p, dim3 grid, int nterms, cudaStream_t s)
{
	int rc = 0;
	if (nterms == 3) {
		rc = adc_smem_optin(scorer_head_kernel<3, NH>, SHCfg<3>::SMEM);
		if (!rc) scorer_head_kernel<3, NH><<<grid, SH_NT, SHCfg<3>::SMEM, s>>>(p);
	} else {
		rc = adc_smem_optin(scorer_head_kernel<1, NH>, SHCfg<1>::SMEM);
		if (!rc) scorer_head_kernel<1, NH><<<grid, SH_NT, SHCfg<1>::SMEM, s>>>(p);
	}
	return rc;
}

// featL / featR: (fm, H, W) tower outputs of the left / right image; volL / volR: (D, H, W), either may be NULL.  Entries
// with x - d < 0 (volL) / x + d >= W (volR) are NOT written (the caller pre-fills NaN like main.lua:962, and applies
// fix_border afterwards, :981).  nterms: 3 = bf16 split (fp32-grade, default), 1 = plain bf16.
extern "C" int mccnn_scorer_head_forward(const mccnn_scorer_head *h, const float *featL, const float *featR, float *volL, float *volR,
					  int H, int W, int D, int nterms, adcensus_stream_t stream)
{
	if (!h || !featL || !featR || (!volL && !volR) || H < 1 || W < 1 || D < 1 || (nterms != 1 && nterms != 3)) return ADCENSUS_EINVAL;
	if (H > 65535) return ADCENSUS_ELIMIT;
	SHParams p;
	memset(&p, 0, sizeof(p));
	p.featL = featL; p.featR = featR; p.volL = volL; p.volR = volR;
	p.wslabs = h->wslabs; p.consts = h->consts;
	for (int l = 0; l < h->l2; l++) {
		p.slab_off[l] = h->slab_off[l];
		p.nk[l] = h->nk[l];
	}
	p.fm = h->fm; p.N = h->nh2; p.L = h->l2; p.H = H; p.W = W; p.D = D;
	cudaStream_t s = adc_stream(stream);
	const dim3 grid(adc_div_up(W, SH_M), H);
	int rc;
	switch (h->nh2) {
	case 128: rc = sh_launch<64>(p, grid, nterms, s); break;
	case 256: rc = sh_launch<128>(p, grid, nterms, s); break;
	case 384: rc = sh_launch<192>(p, grid, nterms, s); break;
	default: return ADCENSUS_ELIMIT;
	}
	if (rc) return rc;
	ADC_CHECK_LAUNCH();
	return 0;
}
