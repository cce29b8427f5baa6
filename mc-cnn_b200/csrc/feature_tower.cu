// feature_tower.cu -- the feature tower of mc-cnn in-library: l1 x [3x3 convolution, stride 1, zero pad 1]
// with ReLU between the layers (and after the last one for the accurate architecture), optionally followed by Normalize2
// (adcensus.cu:1284-1308: x / sqrt(sum_c x^2 + 1e-5)) -- the producer of StereoJoin's inputs (main.lua:726-749, 897-901,
// 944-951; for arch 'slow' main.lua:682-686).  The reference runs cudnn.SpatialConvolution modules (cross-correlation, no
// kernel flip) with cudnn.benchmark picking the algorithm.
//
// Layer 1 has 1 (grey) or 3 input planes: 9..27 multiply-adds per output, done exactly in fp32 on the CUDA cores.
// Layers 2.. (Cin = fm = 64 / 112) are an implicit GEMM on the tensor cores with the machinery of scorer_head.cu:
//   * tile = 128 consecutive pixels of one image row, two warpgroups of 64 rows (wgmma M), N = fm output planes (padded to
//     a multiple of 64), K = 9 Cin ordered tap-major (k = tap * Cin + c), wgmma m64nNk16 with bf16-SPLIT operands (three
//     MMAs per K step: hi.whi + lo.whi + hi.wlo, fp32 accumulation in registers) => fp32-grade results (~1e-6 relative);
//   * the A operand is built in shared memory by eight warps straight from the (Cin, H, W) activation (coalesced along x,
//     zero outside the image), a few taps at a time (K <= 320 per pass: 164 KB for hi + lo), the passes accumulate into the
//     same accumulator;
//   * weights are pre-split into per-K-step slabs and stream from L2 through a 12-slot cp.async.bulk ring;
//   * epilogue straight from the accumulator fragment (a thread holds two pixels x 2 planes per 8 planes); + bias, ReLU, and
//     for the last layer of the fast architecture the Normalize2 of Normalize2.lua fused in (per-pixel sum of squares over the
//     planes, reduced over the four threads sharing the pixel), stores of 8 consecutive pixels per plane and thread quad.
#include <stdlib.h>
#include <string.h>

#include "wgmma.cuh"

namespace {

constexpr int SH_M = 128;                          // pixels per tile
constexpr int SH_ACHUNK = SH_M * 16;               // one 8-wide K chunk of an A operand: [128 rows][8 bf16]
constexpr int FT_KA = 320;                         // K of one pass (A operand capacity)
constexpr int FT_ABYTES = (FT_KA / 8) * SH_ACHUNK; // 81920 per hi / lo
constexpr int FT_NMAX = 128, FT_LMAX = 8;
constexpr int FT_SLAB = 2 * FT_NMAX * 16;          // 4096: one K = 16 step of B at N = 128
constexpr int FT_NSLOT = 12;
constexpr int FT_NCONS = 256, FT_NT = FT_NCONS + 32;   // two consumer warpgroups + weight producer warp
constexpr int FT_OFF_AHI = 0, FT_OFF_ALO = FT_ABYTES, FT_OFF_RING = 2 * FT_ABYTES;
constexpr int FT_OFF_BIAS = FT_OFF_RING + FT_NSLOT * FT_SLAB;
constexpr int FT_OFF_BAR = FT_OFF_BIAS + FT_NMAX * 4;
constexpr int FT_SMEM = FT_OFF_BAR + 2 * FT_NSLOT * 8;
static_assert(FT_SMEM <= 232448, "shared memory budget");

struct FTParams {
	const float *in;                 // (nimg, Cin, H, W)
	float *out;                      // (nimg, fm, H, W)
	const unsigned char *wslabs;     // per K step: [hi slab][lo slab], slab = [2][Np][8] bf16, k = tap * Cin + c
	const float *bias;               // [fm]
	int Cin, fm, Np, H, W, relu, normalize, taps_per_pass;
};

// epilogue of one warpgroup's 64 x NP accumulator block: rows r0, r0 + 8 of pixels x0 + (row), planes 8 j + 2 q (+1)
template <int NP>
__device__ __forceinline__ void ft_epilogue(const FTParams &p, const float (&acc)[NP / 2], const float *bias, float *dst_img, int y,
					    int xa, int xb, int q)
{
	const long HW = (long)p.H * p.W;
	float z[NP / 2];
#pragma unroll
	for (int i = 0; i < NP / 2; i++) {
		const int c = 8 * (i >> 2) + 2 * q + (i & 1);
		z[i] = acc[i] + bias[c];
		if (p.relu) z[i] = fmaxf(z[i], 0.0f);
	}
	if (p.normalize) {
		float sa = 0.0f, sb = 0.0f;
#pragma unroll
		for (int i = 0; i < NP / 2; i++) {
			const int c = 8 * (i >> 2) + 2 * q + (i & 1);
			if (c < p.fm) {
				if (i & 2) sb = fmaf(z[i], z[i], sb);
				else sa = fmaf(z[i], z[i], sa);
			}
		}
		sa += __shfl_xor_sync(0xffffffffu, sa, 1);
		sb += __shfl_xor_sync(0xffffffffu, sb, 1);
		sa += __shfl_xor_sync(0xffffffffu, sa, 2);
		sb += __shfl_xor_sync(0xffffffffu, sb, 2);
		const float ka = sqrtf(sa + 1e-5f), kb = sqrtf(sb + 1e-5f);                // adcensus.cu:1293-1305
#pragma unroll
		for (int i = 0; i < NP / 2; i++) z[i] = z[i] / ((i & 2) ? kb : ka);
	}
	const int W = p.W;
	float *da = dst_img + (long)y * W + xa, *db = dst_img + (long)y * W + xb;
#pragma unroll
	for (int i = 0; i < NP / 2; i++) {
		const int c = 8 * (i >> 2) + 2 * q + (i & 1);
		if (c < p.fm) {
			if (i & 2) {
				if (xb < W) db[(long)c * HW] = z[i];
			} else {
				if (xa < W) da[(long)c * HW] = z[i];
			}
		}
	}
}

template <int NTERMS, int NP>
__global__ void __launch_bounds__(FT_NT, 1)
conv3x3_wgmma_kernel(const FTParams p)
{
	extern __shared__ __align__(128) unsigned char ft_smem[];
	unsigned char *a_hi = ft_smem + FT_OFF_AHI, *a_lo = ft_smem + FT_OFF_ALO, *ring = ft_smem + FT_OFF_RING;
	float *bias = reinterpret_cast<float *>(ft_smem + FT_OFF_BIAS);
	uint64_t *bar_full = reinterpret_cast<uint64_t *>(ft_smem + FT_OFF_BAR);
	uint64_t *bar_empty = bar_full + FT_NSLOT;

	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int x0 = blockIdx.x * SH_M, y = blockIdx.y, img = blockIdx.z;
	const int Cin = p.Cin, H = p.H, W = p.W;
	const long HW = (long)H * W;
	const int npass = (9 + p.taps_per_pass - 1) / p.taps_per_pass;
	const uint32_t slab_bytes = (uint32_t)NP * 32u;

	if (tid == 0) {
		for (int s = 0; s < FT_NSLOT; s++) {
			mbar_init(&bar_full[s], 1);
			mbar_init(&bar_empty[s], 2);           // one arrival per consumer warpgroup
		}
		mbar_fence_init();
	}
	for (int i = tid; i < FT_NMAX; i += FT_NT) bias[i] = i < p.fm ? p.bias[i] : 0.0f;
	__syncthreads();

	if (warp == 8) {
		// ------------------------------------------------------------ weight producer: every K step of the layer, in order
		if (lane == 0) {
			const int nks = 9 * Cin / 16;
			for (unsigned it = 0; it < (unsigned)(nks * (NTERMS == 3 ? 2 : 1)); it++) {
				const int s = it % FT_NSLOT;
				const int ks = NTERMS == 3 ? it >> 1 : it, part = NTERMS == 3 ? it & 1 : 0;
				if (it >= (unsigned)FT_NSLOT) sh_wait(&bar_empty[s], ((it / FT_NSLOT) - 1) & 1);
				mbar_arrive_expect_tx(&bar_full[s], slab_bytes);
				sh_bulk_load(ring + s * FT_SLAB, p.wslabs + ((long)ks * 2 + part) * slab_bytes, slab_bytes, &bar_full[s]);
			}
		}
		return;
	}
	// ---------------------------------------------------------------- consumers: build the operand (all 256 threads), MMAs and
	// epilogue per warpgroup (warpgroup g: rows 64 g .. 64 g + 63 of the tile)
	const int m = (warp & 3) * 32 + lane, hf = warp >> 2;
	const int x = x0 + m;
	const int g = tid >> 7, t = tid & 127;
	const int r0 = 64 * g + 16 * (t >> 5) + (lane >> 2), q = lane & 3;
	const float *src_img = p.in + (long)img * Cin * HW;
	const uint32_t a_hi_s = tma_smem_addr(a_hi) + g * 64 * 16, a_lo_s = tma_smem_addr(a_lo) + g * 64 * 16, ring_s = tma_smem_addr(ring);
	const uint32_t lbo_b = (uint32_t)NP * 16u;
	float acc[NP / 2];
#pragma unroll
	for (int i = 0; i < NP / 2; i++) acc[i] = 0.0f;
	unsigned it = 0;
	int tap0 = 0;
	for (int ps = 0; ps < npass; ps++) {
		const int ntap = min(p.taps_per_pass, 9 - tap0);
		const int nch = ntap * Cin / 8;                       // 8-wide K chunks of this pass
		if (ps > 0) sh_bar(1, FT_NCONS);                      // both warpgroups' MMAs of the previous pass have read the operand
		// chunk kc: tap = tap0 + (8 kc) / Cin, planes c0 .. c0 + 7 (Cin % 8 == 0: a chunk never straddles a tap)
		for (int kc0 = hf * 4; kc0 < nch; kc0 += 8) {          // each half takes alternate groups of 4 chunks
			float v[4][8];
#pragma unroll
			for (int u = 0; u < 4; u++) {
				const int kc = kc0 + u;
				const int k0 = kc * 8, tap = tap0 + k0 / Cin, c0 = k0 % Cin;
				const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
				const bool ok = kc < nch && yy >= 0 && yy < H && xx >= 0 && xx < W;
				const float *src = src_img + (long)c0 * HW + (long)(ok ? yy : 0) * W + (ok ? xx : 0);
#pragma unroll
				for (int e = 0; e < 8; e++) v[u][e] = ok ? __ldg(src + (long)e * HW) : 0.0f;
			}
#pragma unroll
			for (int u = 0; u < 4; u++)
				if (kc0 + u < nch) sh_store8<NTERMS>(a_hi, a_lo, SH_ACHUNK, kc0 + u, m, v[u]);
		}
		fence_proxy_async_smem();
		sh_bar(1, FT_NCONS);
		wg_fence_acc(acc);
		wg_fence();
		int pend = -1;
		for (int ks = 0; ks < nch / 2; ks++) {
			const uint64_t da_hi = sh_desc(a_hi_s + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
			const uint64_t da_lo = sh_desc(a_lo_s + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
#pragma unroll
			for (int part = 0; part < (NTERMS == 3 ? 2 : 1); part++, it++) {
				const int s = it % FT_NSLOT;
				sh_wait_mma(&bar_full[s], (it / FT_NSLOT) & 1);
				const uint64_t db = sh_desc(ring_s + s * FT_SLAB, lbo_b, 128);
				if (part == 0) {
					wg_mma<NP>(acc, da_hi, db, (ps > 0 || ks > 0) ? 1u : 0u);
					if (NTERMS == 3) wg_mma<NP>(acc, da_lo, db, 1);
				} else {
					wg_mma<NP>(acc, da_hi, db, 1);
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
		tap0 += ntap;
	}
	ft_epilogue<NP>(p, acc, bias, p.out + (long)img * p.fm * HW, y, x0 + r0, x0 + r0 + 8, q);
}

// ---- second form, for Cin = fm <= 64 (the fast architecture): weights RESIDENT, persistent CTAs --------------------------
// With 64 planes the whole layer's weights, split, are 147 KB: they stay in shared memory for the life of a persistent CTA; the
// A operand is built one TAP at a time (K = 64: 32 KB for hi + lo) into a double buffer, so the eight builder warps (next
// tap's loads already in flight while the current one is split and stored) and the two MMA / epilogue warpgroups overlap.
constexpr int F2_NB = 256, F2_NC = 256, F2_NT = F2_NB + F2_NC;           // builders, consumer warpgroups
constexpr int F2_WBYTES = 9 * 64 / 16 * 2 * 64 * 32;                       // 147456: 36 K steps x (hi, lo) x [2][64][8] bf16
constexpr int F2_ABUF = 2 * (64 / 8) * SH_ACHUNK;                         // one tap: hi + lo = 32768
constexpr int F2_OFF_A = F2_WBYTES, F2_OFF_BIAS = F2_OFF_A + 2 * F2_ABUF;
constexpr int F2_OFF_BAR = F2_OFF_BIAS + 64 * 4;                           // a_full[2], a_free[2]
constexpr int F2_SMEM = F2_OFF_BAR + 4 * 8;
static_assert(F2_SMEM <= 232448, "shared memory budget");

template <int NTERMS>
__global__ void __launch_bounds__(F2_NT, 1)
conv3x3_resident_kernel(const FTParams p, int nimg)
{
	extern __shared__ __align__(128) unsigned char ft_smem[];
	unsigned char *wsm = ft_smem, *abuf = ft_smem + F2_OFF_A;
	float *bias = reinterpret_cast<float *>(ft_smem + F2_OFF_BIAS);
	uint64_t *a_full = reinterpret_cast<uint64_t *>(ft_smem + F2_OFF_BAR), *a_free = a_full + 2;

	const int tid = threadIdx.x, lane = tid & 31;
	const int H = p.H, W = p.W, Cin = p.Cin;                      // Cin == 64, Np == 64
	const long HW = (long)H * W;
	const int xt = (W + SH_M - 1) / SH_M;
	const int ntile = nimg * H * xt;
	const int nks_tap = Cin / 16;
	const uint32_t slab = 64u * 32u;

	if (tid == 0) {
		for (int i = 0; i < 2; i++) {
			mbar_init(&a_full[i], F2_NB);
			mbar_init(&a_free[i], 2);                          // one arrival per consumer warpgroup
		}
		mbar_fence_init();
	}
	{   // the layer's weights: a straight copy of the prepared slabs
		const uint4 *src = reinterpret_cast<const uint4 *>(p.wslabs);
		uint4 *dst = reinterpret_cast<uint4 *>(wsm);
		const int n16 = 9 * nks_tap * 2 * (int)slab / 16;
		for (int i = tid; i < n16; i += F2_NT) dst[i] = __ldg(src + i);
	}
	for (int i = tid; i < 64; i += F2_NT) bias[i] = i < p.fm ? p.bias[i] : 0.0f;
	fence_proxy_async_smem();                                  // the weights were written with generic stores
	__syncthreads();

	if (tid < F2_NB) {
		// ------------------------------------------------------------ operand builders: thread = (pixel m, 4 of the tap's 8 chunks)
		const int m = tid & 127, hf = tid >> 7;
		float nxt[4][8];
		auto load = [&](int tile, int tap, float (&v)[4][8]) {
			const int img = tile / (H * xt), rem = tile - img * (H * xt), y = rem / xt, x = (rem - y * xt) * SH_M + m;
			const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
			const bool ok = tile < ntile && yy >= 0 && yy < H && xx >= 0 && xx < W;
			const float *src = p.in + (long)img * Cin * HW + (long)(hf * 32) * HW + (long)(ok ? yy : 0) * W + (ok ? xx : 0);
#pragma unroll
			for (int u = 0; u < 4; u++)
#pragma unroll
				for (int e = 0; e < 8; e++) v[u][e] = ok ? __ldg(src + (long)(u * 8 + e) * HW) : 0.0f;
		};
		unsigned g = 0;
		int tile = blockIdx.x, tap = 0;
		if (tile < ntile) load(tile, 0, nxt);
		while (tile < ntile) {
			float cur[4][8];
#pragma unroll
			for (int u = 0; u < 4; u++)
#pragma unroll
				for (int e = 0; e < 8; e++) cur[u][e] = nxt[u][e];
			int ntile_i = tile, ntap = tap + 1;                 // the step after this one
			if (ntap == 9) { ntap = 0; ntile_i = tile + gridDim.x; }
			load(ntile_i, ntap, nxt);                           // in flight while this step is split and stored
			const int b = g & 1;
			if (g >= 2) sh_wait(&a_free[b], ((g >> 1) - 1) & 1);
			unsigned char *ah = abuf + b * F2_ABUF, *al = ah + (64 / 8) * SH_ACHUNK;
#pragma unroll
			for (int u = 0; u < 4; u++) sh_store8<NTERMS>(ah, al, SH_ACHUNK, hf * 4 + u, m, cur[u]);
			fence_proxy_async_smem();
			sh_arrive(&a_full[b]);
			g++;
			tile = ntile_i;
			tap = ntap;
		}
	} else {
		// ------------------------------------------------------------ consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of each tile
		const int c = tid - F2_NB, wg = c >> 7, t = c & 127;
		const int r0 = 64 * wg + 16 * (t >> 5) + (lane >> 2), q = lane & 3;
		const uint32_t a_s = tma_smem_addr(abuf) + wg * 64 * 16, w_s = tma_smem_addr(wsm);
		const uint32_t lbo_b = 64u * 16u;
		float acc[32];
#pragma unroll
		for (int i = 0; i < 32; i++) acc[i] = 0.0f;
		unsigned g = 0;
		for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
			const int img = tile / (H * xt), rem = tile - img * (H * xt), y = rem / xt, x0 = (rem - y * xt) * SH_M;
			wg_fence_acc(acc);
			int pend = -1;
			for (int tap = 0; tap < 9; tap++, g++) {
				const int b = g & 1;
				sh_wait(&a_full[b], (g >> 1) & 1);
				wg_fence();
#pragma unroll
				for (int ks = 0; ks < 4; ks++) {
					const uint64_t da_hi = sh_desc(a_s + b * F2_ABUF + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
					const uint64_t da_lo = sh_desc(a_s + b * F2_ABUF + (64 / 8) * SH_ACHUNK + ks * 2 * SH_ACHUNK, SH_ACHUNK, 128);
					const uint32_t wk = w_s + (uint32_t)(tap * nks_tap + ks) * 2u * slab;
					const uint64_t db_hi = sh_desc(wk, lbo_b, 128), db_lo = sh_desc(wk + slab, lbo_b, 128);
					wg_mma<64>(acc, da_hi, db_hi, (tap > 0 || ks > 0) ? 1u : 0u);
					if (NTERMS == 3) {
						wg_mma<64>(acc, da_lo, db_hi, 1);
						wg_mma<64>(acc, da_hi, db_lo, 1);
					}
				}
				wg_commit();
				wg_wait<1>();                                   // the previous tap's MMAs are done: its buffer is free
				if (pend >= 0 && t == 0) sh_arrive(&a_free[pend]);
				pend = b;
			}
			wg_wait<0>();
			wg_fence_acc(acc);
			if (t == 0) sh_arrive(&a_free[pend]);
			ft_epilogue<64>(p, acc, bias, p.out + (long)img * p.fm * HW, y, x0 + r0, x0 + r0 + 8, q);
		}
	}
}

// first layer (Cin = 1 or 3): exact fp32, thread = pixel, weights in shared memory; planes / rows / columns ascending
__global__ void conv3x3_first_kernel(const float *__restrict__ in, const float *__restrict__ w, const float *__restrict__ b,
				     float *__restrict__ out, int Cin, int fm, int H, int W, int relu)
{
	extern __shared__ float fw[];                         // [fm][Cin * 9] + [fm]
	const int nw = fm * Cin * 9;
	for (int i = threadIdx.x; i < nw + fm; i += blockDim.x) fw[i] = i < nw ? w[i] : b[i - nw];
	__syncthreads();
	const long HW = (long)H * W;
	const long id = (long)blockIdx.x * blockDim.x + threadIdx.x;
	const int img = blockIdx.y;
	if (id >= HW) return;
	const int y = (int)(id / W), x = (int)(id % W);
	float v[27];
	for (int c = 0; c < Cin; c++)
#pragma unroll
		for (int t = 0; t < 9; t++) {
			const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
			v[c * 9 + t] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? in[((long)img * Cin + c) * HW + (long)yy * W + xx] : 0.0f;
		}
	float *dst = out + (long)img * fm * HW + id;
	for (int o = 0; o < fm; o++) {
		float acc = fw[nw + o];
		for (int k = 0; k < Cin * 9; k++) acc = fmaf(fw[o * Cin * 9 + k], v[k], acc);
		dst[(long)o * HW] = relu ? fmaxf(acc, 0.0f) : acc;
	}
}

// weights (fm, Cin, 3, 3) fp32 -> slabs over k = tap * Cin + c: per K step [hi: [2][Np][8] bf16][lo: ...], planes >= fm zero
__global__ void ft_prep_kernel(const float *__restrict__ w, unsigned short *__restrict__ slabs, int fm, int Np, int Cin)
{
	const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (long)fm * Cin * 9) return;
	const int o = (int)(i / (Cin * 9)), c = (int)((i / 9) % Cin), tap = (int)(i % 9);
	const int k = tap * Cin + c;
	const float v = w[i];
	const unsigned hb = __float_as_uint(v);
	const unsigned hi = (hb + 0x7fffu + ((hb >> 16) & 1u)) >> 16;
	const float r = v - __uint_as_float(hi << 16);
	const unsigned rb = __float_as_uint(r);
	const unsigned lo = (rb + 0x7fffu + ((rb >> 16) & 1u)) >> 16;
	const int ks = k / 16, j = (k / 8) & 1, e = k & 7;
	const long slab = (long)Np * 16;
	const long base = (long)ks * 2 * slab + ((long)j * Np + o) * 8 + e;
	slabs[base] = (unsigned short)hi;
	slabs[base + slab] = (unsigned short)lo;
}

}  // namespace

struct mccnn_feature_tower {
	int n_in, fm, Np, l1, relu_last, normalize, device;
	float *w0, *b0;                     // first layer
	unsigned char *wslabs[FT_LMAX];     // layers 1 .. l1-1
	float *bias[FT_LMAX];
};

// W[i] (fm, cin_i, 3, 3) row-major / b[i] (fm) for i = 0 .. l1-1, DEVICE pointers, the layout of cudnn.SpatialConvolution's
// weight / bias (main.lua:683, 729).  n_in = 1 or 3 input planes; relu_last / normalize: arch 'fast' = (0, 1), 'slow' = (1, 0).
extern "C" int mccnn_feature_tower_create(mccnn_feature_tower **out, int n_in, int fm, int l1, int relu_last, int normalize,
					   const float *const *W, const float *const *b, int device, adcensus_stream_t stream)
{
	if (!out || !W || !b || (n_in != 1 && n_in != 3) || fm < 8 || l1 < 1) return ADCENSUS_EINVAL;
	if (l1 > FT_LMAX || fm > FT_NMAX || (fm % 16)) return ADCENSUS_ELIMIT;
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(device);
	cudaStream_t s = adc_stream(stream);
	mccnn_feature_tower *h = (mccnn_feature_tower *)calloc(1, sizeof(*h));
	if (!h) return ADCENSUS_EINVAL;
	h->n_in = n_in; h->fm = fm; h->Np = (fm + 63) / 64 * 64; h->l1 = l1; h->relu_last = relu_last; h->normalize = normalize; h->device = device;
	int rc = (int)cudaMalloc((void **)&h->w0, (size_t)fm * n_in * 9 * sizeof(float));
	if (!rc) rc = (int)cudaMalloc((void **)&h->b0, fm * sizeof(float));
	if (!rc) rc = (int)cudaMemcpyAsync(h->w0, W[0], (size_t)fm * n_in * 9 * sizeof(float), cudaMemcpyDeviceToDevice, s);
	if (!rc) rc = (int)cudaMemcpyAsync(h->b0, b[0], fm * sizeof(float), cudaMemcpyDeviceToDevice, s);
	for (int l = 1; l < l1 && !rc; l++) {
		const size_t bytes = (size_t)(9 * fm / 16) * 2 * h->Np * 32;
		rc = (int)cudaMalloc((void **)&h->wslabs[l], bytes);
		if (!rc) rc = (int)cudaMemsetAsync(h->wslabs[l], 0, bytes, s);
		if (!rc) rc = (int)cudaMalloc((void **)&h->bias[l], fm * sizeof(float));
		if (!rc) rc = (int)cudaMemcpyAsync(h->bias[l], b[l], fm * sizeof(float), cudaMemcpyDeviceToDevice, s);
		if (!rc) {
			ft_prep_kernel<<<adc_div_up((long)fm * fm * 9, 256), 256, 0, s>>>(W[l], (unsigned short *)h->wslabs[l], fm, h->Np, fm);
			rc = (int)cudaPeekAtLastError();
		}
	}
	if (!rc) rc = (int)cudaStreamSynchronize(s);
	cudaSetDevice(prev);
	if (rc) {
		*out = nullptr;
		for (int l = 0; l < FT_LMAX; l++) { cudaFree(h->wslabs[l]); cudaFree(h->bias[l]); }
		cudaFree(h->w0); cudaFree(h->b0);
		free(h);
		return rc;
	}
	*out = h;
	return 0;
}

extern "C" void mccnn_feature_tower_destroy(mccnn_feature_tower *h)
{
	if (!h) return;
	for (int l = 0; l < FT_LMAX; l++) { cudaFree(h->wslabs[l]); cudaFree(h->bias[l]); }
	cudaFree(h->w0); cudaFree(h->b0);
	free(h);
}

template <int NTERMS>
static void ft_launch(const FTParams &p, dim3 grid, cudaStream_t s)
{
	if (p.Np == 64)
		conv3x3_wgmma_kernel<NTERMS, 64><<<grid, FT_NT, FT_SMEM, s>>>(p);
	else
		conv3x3_wgmma_kernel<NTERMS, 128><<<grid, FT_NT, FT_SMEM, s>>>(p);
}

// img (nimg, n_in, H, W) -> out (nimg, fm, H, W); nimg = 2 for a stereo pair (x_batch of main.lua:944).  nterms: 3 = bf16-split
// operands (fp32-grade), 1 = plain bf16.  Intermediate activations live in stream-ordered scratch.
extern "C" int mccnn_feature_tower_forward(const mccnn_feature_tower *h, const float *img, float *out, int nimg, int H, int W,
					    int nterms, adcensus_stream_t stream)
{
	if (!h || !img || !out || nimg < 1 || H < 1 || W < 1 || (nterms != 1 && nterms != 3)) return ADCENSUS_EINVAL;
	if (H > 65535 || nimg > 65535) return ADCENSUS_ELIMIT;
	cudaStream_t s = adc_stream(stream);
	const long HW = (long)H * W;
	const size_t act = (size_t)nimg * h->fm * HW * sizeof(float);
	float *buf[2] = {nullptr, nullptr};
	int rc = 0;
	if (h->l1 > 1) rc = adc_scratch_alloc((void **)&buf[0], act, s);
	if (!rc && h->l1 > 2) rc = adc_scratch_alloc((void **)&buf[1], act, s);
	if (rc) return rc;
	// layer 1
	{
		float *dst = h->l1 == 1 ? out : buf[0];
		const int relu = h->l1 > 1 ? 1 : h->relu_last;
		const dim3 grid(adc_div_up(HW, 128), nimg);
		const size_t sm = (size_t)(h->fm * h->n_in * 9 + h->fm) * sizeof(float);
		conv3x3_first_kernel<<<grid, 128, sm, s>>>(img, h->w0, h->b0, dst, h->n_in, h->fm, H, W, relu);
		rc = (int)cudaPeekAtLastError();
	}
	for (int l = 1; l < h->l1 && !rc; l++) {
		const bool last = l + 1 == h->l1;
		FTParams p;
		memset(&p, 0, sizeof(p));
		p.in = buf[(l - 1) & 1];
		p.out = last ? out : buf[l & 1];
		p.wslabs = h->wslabs[l]; p.bias = h->bias[l];
		p.Cin = h->fm; p.fm = h->fm; p.Np = h->Np; p.H = H; p.W = W;
		p.relu = last ? h->relu_last : 1;
		p.normalize = last ? h->normalize : 0;
		p.taps_per_pass = FT_KA / h->fm;                       // K of a pass = taps x Cin <= 320
		if (p.taps_per_pass > 9) p.taps_per_pass = 9;
		const dim3 grid(adc_div_up(W, SH_M), H, nimg);
		if (h->fm == 64) {                          // weights resident, persistent CTAs (the fast architecture)
			const int ntile = nimg * H * adc_div_up(W, SH_M);
			const int nb = ntile < adc_num_sms() ? ntile : adc_num_sms();
			if (nterms == 3) {
				rc = adc_smem_optin(conv3x3_resident_kernel<3>, F2_SMEM);
				if (!rc) conv3x3_resident_kernel<3><<<nb, F2_NT, F2_SMEM, s>>>(p, nimg);
			} else {
				rc = adc_smem_optin(conv3x3_resident_kernel<1>, F2_SMEM);
				if (!rc) conv3x3_resident_kernel<1><<<nb, F2_NT, F2_SMEM, s>>>(p, nimg);
			}
			if (!rc) rc = (int)cudaPeekAtLastError();
			continue;
		}
		if (nterms == 3) {
			rc = adc_smem_optin(conv3x3_wgmma_kernel<3, 128>, FT_SMEM);
			if (!rc) rc = adc_smem_optin(conv3x3_wgmma_kernel<3, 64>, FT_SMEM);
			if (!rc) ft_launch<3>(p, grid, s);
		} else {
			rc = adc_smem_optin(conv3x3_wgmma_kernel<1, 128>, FT_SMEM);
			if (!rc) rc = adc_smem_optin(conv3x3_wgmma_kernel<1, 64>, FT_SMEM);
			if (!rc) ft_launch<1>(p, grid, s);
		}
		if (!rc) rc = (int)cudaPeekAtLastError();
	}
	if (h->l1 == 1 && h->normalize && !rc) rc = ADCENSUS_EINVAL;   // a one-layer tower with Normalize2 is not a net of the reference
	for (int i = 0; i < 2; i++)
		if (buf[i]) {
			const int rc2 = adc_scratch_free(buf[i], s);
			if (!rc) rc = rc2;
		}
	return rc;
}
