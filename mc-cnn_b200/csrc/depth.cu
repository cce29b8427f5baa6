// depth.cu -- metric depth, coloured point clouds and depth metrics of a disparity map, for sm_90a (DESIGN §20; an addition
// beyond the reference).
//
// Everything follows one fp32 rule per pixel: a disparity d is valid when it is finite and s = d + doffs (one rounding) is
// > 0; then Z = fB / s, X = ((x - cx) * Z) / f, Y = ((y - cy) * Z) / f, each operation rounded once in that order, fB being
// the host's float64 f * baseline rounded once to fp32.  A numpy float32 restatement gives the same bits.
//
// * mccnn_disp_to_depth: one thread per pixel, NaN where there is no depth.
// * mccnn_point_cloud_count / _fill: the pixels are cut into chunks of CHUNK in row-major order.  count: each block counts
//   its chunk's valid pixels, one block scans the block counts (64-bit, exclusive, in block order) and writes the total.
//   fill: the same two steps, then each block ranks its valid pixels in row-major order (ballots), writes their packed
//   15-byte PLY records into shared memory at the shift of its first global byte modulo 16, and copies them out in aligned
//   16-byte words; only the partial first and last words are written bytewise, so every global byte has one writer.
// * mccnn_depth_metrics: per pixel (the prediction a disparity or already a depth) the integer counts and four float64 terms; each block sums a fixed range of CHUNK pixels
//   in a fixed order, one block adds the block sums in a fixed order: no float atomics, the same bits on every GPU.
// * mccnn_velo_depth_map (DESIGN §21): a LiDAR scan projected into an (H, W) depth map.  The keys are cleared to all ones,
//   each kept point atomicMin-s the 64-bit key (float bits of its z, its index) of its pixel, and one pass decodes the
//   keys.  z > 0, so its bits order like its value: the smallest z wins, the smallest index breaks a tie, and the result
//   does not depend on the order of the atomics.
#include <math.h>

#include <algorithm>

#include "camera.cuh"
#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ITEMS = 8;                         // pixels per thread and chunk
constexpr long CHUNK = (long)THREADS * ITEMS;    // pixels per block
constexpr int REC = 15;                          // bytes per PLY vertex: float x, y, z, uchar r, g, b
constexpr int SCAN_THREADS = 1024;
constexpr unsigned FULL = 0xffffffffu;

__global__ void depth_kernel(const float *__restrict__ disp, long n, int W, Cam c, float *__restrict__ Z, float *__restrict__ X,
			     float *__restrict__ Y)
{
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		float z;
		const bool ok = depth_of(disp[p], c, &z);
		Z[p] = ok ? z : adc_nan();
		if (X) {
			const int y = (int)(p / W), x = (int)(p - (long)y * W);
			X[p] = ok ? lateral(x, c.cx, z, c.f) : adc_nan();
			Y[p] = ok ? lateral(y, c.cy, z, c.f) : adc_nan();
		}
	}
}

// ---- point cloud ----

// valid pixels of chunk blockIdx.x -> blk[blockIdx.x]
__global__ void __launch_bounds__(THREADS) cloud_count_kernel(const float *__restrict__ disp, long n, Cam c, int *__restrict__ blk)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0;
#pragma unroll
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + threadIdx.x;
		float z;
		k += p < n && depth_of(disp[p], c, &z);
	}
	k = __reduce_add_sync(FULL, k);
	if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = k;
	__syncthreads();
	if (threadIdx.x == 0) {
		int t = 0;
		for (int w = 0; w < THREADS / 32; w++) t += warp_n[w];
		blk[blockIdx.x] = t;
	}
}

// off[b] = sum of blk[0 .. b) in 64 bits, *total = the sum of all: each thread scans a contiguous run of blocks
__global__ void __launch_bounds__(SCAN_THREADS) cloud_scan_kernel(const int *__restrict__ blk, int nblk, long long *__restrict__ off,
								    long long *__restrict__ total)
{
	__shared__ long long part[SCAN_THREADS];
	const int per = (nblk + SCAN_THREADS - 1) / SCAN_THREADS;
	const int lo = min(nblk, threadIdx.x * per), hi = min(nblk, lo + per);
	long long s = 0;
	for (int b = lo; b < hi; b++) s += blk[b];
	part[threadIdx.x] = s;
	__syncthreads();
	if (threadIdx.x == 0) {
		long long a = 0;
		for (int t = 0; t < SCAN_THREADS; t++) {
			const long long v = part[t];
			part[t] = a;
			a += v;
		}
		*total = a;
	}
	__syncthreads();
	if (off) {
		s = part[threadIdx.x];
		for (int b = lo; b < hi; b++) {
			off[b] = s;
			s += blk[b];
		}
	}
}

__device__ __forceinline__ void put_float(unsigned char *p, float v)
{
	const unsigned u = __float_as_uint(v);
	p[0] = (unsigned char)u;
	p[1] = (unsigned char)(u >> 8);
	p[2] = (unsigned char)(u >> 16);
	p[3] = (unsigned char)(u >> 24);
}

// the records of chunk blockIdx.x's valid pixels, in row-major order, to out + 15 off[blockIdx.x]; records at or past `cap`
// are dropped
__global__ void __launch_bounds__(THREADS) cloud_fill_kernel(const float *__restrict__ disp, const unsigned char *__restrict__ rgb,
							     int nch, long n, int W, Cam c, const long long *__restrict__ off,
							     unsigned char *__restrict__ out, long long cap)
{
	__shared__ __align__(16) unsigned char sh[CHUNK * REC + 32];
	__shared__ int warp_n[THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const long base = (long)blockIdx.x * CHUNK;
	const long long first = off[blockIdx.x];
	if (first >= cap) return;
	const long long g0 = first * REC;                 // the block's first global byte
	const int shift = (int)(g0 & 15);
	int rank = 0;                                      // records of the chunk's earlier rows of THREADS pixels
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + threadIdx.x;
		float z = 0.f;
		const bool ok = p < n && depth_of(disp[p], c, &z);
		const unsigned m = __ballot_sync(FULL, ok);
		if (lane == 0) warp_n[warp] = __popc(m);
		__syncthreads();
		int before = rank + __popc(m & ((1u << lane) - 1u));
		int all = 0;
		for (int w = 0; w < THREADS / 32; w++) {
			const int v = warp_n[w];
			before += w < warp ? v : 0;
			all += v;
		}
		if (ok) {
			const int y = (int)(p / W), x = (int)(p - (long)y * W);
			unsigned char *r = sh + shift + before * REC;
			put_float(r, lateral(x, c.cx, z, c.f));
			put_float(r + 4, lateral(y, c.cy, z, c.f));
			put_float(r + 8, z);
			if (nch == 3) {
				r[12] = rgb[3 * p];
				r[13] = rgb[3 * p + 1];
				r[14] = rgb[3 * p + 2];
			} else {
				r[12] = r[13] = r[14] = rgb[p];
			}
		}
		rank += all;
		__syncthreads();                           // warp_n is rewritten by the next row
	}
	const long long kept = min((long long)rank, cap - first);
	const long long g1 = g0 + kept * REC;          // one past the block's last global byte
	const long long a0 = g0 - shift;               // 16-byte aligned; sh[0] stands for out[a0]
	const int nwords = (int)((g1 - a0 + 15) >> 4);
	for (int w = threadIdx.x; w < nwords; w += THREADS) {
		const long long g = a0 + 16ll * w;
		if (g >= g0 && g + 16 <= g1) {
			*reinterpret_cast<uint4 *>(out + g) = *reinterpret_cast<const uint4 *>(sh + 16 * w);
		} else {
			for (int b = 0; b < 16; b++)
				if (g + b >= g0 && g + b < g1) out[g + b] = sh[16 * w + b];
		}
	}
}

// block counts, then their scan: off (nblk) may be NULL when only the total is wanted
int cloud_scan(const float *disp, long n, const Cam &c, int *blk, long long *off, long long *total, cudaStream_t s)
{
	const int nblk = adc_div_up(n, CHUNK);
	cloud_count_kernel<<<nblk, THREADS, 0, s>>>(disp, n, c, blk);
	ADC_CHECK_LAUNCH();
	cloud_scan_kernel<<<1, SCAN_THREADS, 0, s>>>(blk, nblk, off, total);
	ADC_CHECK_LAUNCH();
	return 0;
}

// ---- depth metrics ----

constexpr int NSUM = 4;  // abs_rel, sq_rel, squared error, squared log error

__device__ __forceinline__ float clampf(float z, float lo, float hi) { return z < lo ? lo : (z > hi ? hi : z); }

// the counts of chunk blockIdx.x added to counts (integer atomics); its NSUM float64 sums to part[NSUM blockIdx.x + k]
__global__ void __launch_bounds__(THREADS) metrics_kernel(const float *__restrict__ pred, int pred_depth, const float *__restrict__ gt,
							  long n, Cam c, float min_depth, unsigned long long *__restrict__ counts,
							  double *__restrict__ part)
{
	__shared__ unsigned block_counts[MCCNN_DEPTH_NCOUNT];
	__shared__ double sh[NSUM][THREADS];
	const int tid = threadIdx.x;
	if (tid < MCCNN_DEPTH_NCOUNT) block_counts[tid] = 0;
	unsigned k[MCCNN_DEPTH_NCOUNT];
#pragma unroll
	for (int j = 0; j < MCCNN_DEPTH_NCOUNT; j++) k[j] = 0;
	double s[NSUM] = {0.0, 0.0, 0.0, 0.0};
	Cam open = c;
	open.max_depth = CUDART_INF_F;                 // validity without the cap; the range test and the clamp follow
	const long base = (long)blockIdx.x * CHUNK;
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + tid;
		if (p >= n) break;
		float zg, zp;
		if (!depth_of(gt[p], open, &zg) || !(zg >= min_depth && zg <= c.max_depth)) continue;
		k[MCCNN_DEPTH_GT]++;
		zp = pred[p];
		if (pred_depth ? !(isfinite(zp) && zp > 0.f) : !depth_of(zp, open, &zp)) continue;
		zp = clampf(zp, min_depth, c.max_depth);
		const double a = zp, b = zg, e = __dsub_rn(a, b), e2 = __dmul_rn(e, e);
		const double l = __dsub_rn(log(a), log(b));
		const double r = fmax(__ddiv_rn(a, b), __ddiv_rn(b, a));
		k[MCCNN_DEPTH_N]++;
		k[MCCNN_DEPTH_A1] += r < 1.25;
		k[MCCNN_DEPTH_A2] += r < 1.25 * 1.25;
		k[MCCNN_DEPTH_A3] += r < 1.25 * 1.25 * 1.25;
		s[0] = __dadd_rn(s[0], __ddiv_rn(fabs(e), b));
		s[1] = __dadd_rn(s[1], __ddiv_rn(e2, b));
		s[2] = __dadd_rn(s[2], e2);
		s[3] = __dadd_rn(s[3], __dmul_rn(l, l));
	}
	__syncthreads();                               // block_counts zeroed
#pragma unroll
	for (int j = 0; j < MCCNN_DEPTH_NCOUNT; j++) {
		const unsigned w = __reduce_add_sync(FULL, k[j]);
		if ((tid & 31) == 0 && w) atomicAdd(&block_counts[j], w);
	}
#pragma unroll
	for (int j = 0; j < NSUM; j++) sh[j][tid] = s[j];
	__syncthreads();
	if (tid < MCCNN_DEPTH_NCOUNT && block_counts[tid]) atomicAdd(counts + tid, (unsigned long long)block_counts[tid]);
	for (int h = THREADS / 2; h; h >>= 1) {        // a fixed tree
		if (tid < h)
#pragma unroll
			for (int j = 0; j < NSUM; j++) sh[j][tid] = __dadd_rn(sh[j][tid], sh[j][tid + h]);
		__syncthreads();
	}
	if (tid < NSUM) part[NSUM * blockIdx.x + tid] = sh[tid][0];
}

// sums[k] = the block sums added in a fixed order: thread t over blocks t, t + THREADS, ..., then a tree
__global__ void __launch_bounds__(THREADS) metrics_finish_kernel(const double *__restrict__ part, int nblk, double *__restrict__ sums)
{
	__shared__ double sh[NSUM][THREADS];
	const int tid = threadIdx.x;
	double a[NSUM] = {0.0, 0.0, 0.0, 0.0};
	for (int b = tid; b < nblk; b += THREADS)
#pragma unroll
		for (int j = 0; j < NSUM; j++) a[j] = __dadd_rn(a[j], part[NSUM * b + j]);
#pragma unroll
	for (int j = 0; j < NSUM; j++) sh[j][tid] = a[j];
	__syncthreads();
	for (int h = THREADS / 2; h; h >>= 1) {
		if (tid < h)
#pragma unroll
			for (int j = 0; j < NSUM; j++) sh[j][tid] = __dadd_rn(sh[j][tid], sh[j][tid + h]);
		__syncthreads();
	}
	if (tid < NSUM) sums[tid] = sh[tid][0];
}

// ---- LiDAR scans projected into a sparse depth map (DESIGN §21) ----

constexpr unsigned long long NO_POINT = ~0ull;   // every key's high word is a finite float's bits, never all ones

struct Proj {
	float p[12];                                   // row-major 3x4
};

// r . (x, y, z, 1) in fp32, each operation rounded once, left to right
__device__ __forceinline__ float proj_row(const float *r, float x, float y, float z)
{
	return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z)), r[3]);
}

// each point's key (z bits << 32 | index) min-ed into the key of its pixel
__global__ void velo_key_kernel(const float4 *__restrict__ pts, long long n, Proj P, int H, int W, float min_depth,
				unsigned long long *__restrict__ key)
{
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		const float4 q = pts[i];
		const float z = proj_row(P.p + 8, q.x, q.y, q.z);
		if (!(z > min_depth && z < CUDART_INF_F)) continue;
		const float fu = rintf(__fdiv_rn(proj_row(P.p, q.x, q.y, q.z), z));
		const float fv = rintf(__fdiv_rn(proj_row(P.p + 4, q.x, q.y, q.z), z));
		if (!(fu >= 1.f && fu <= (float)W && fv >= 1.f && fv <= (float)H)) continue;
		const long p = (long)((int)fv - 1) * W + ((int)fu - 1);
		atomicMin(key + p, (unsigned long long)__float_as_uint(z) << 32 | (unsigned long long)i);
	}
}

__global__ void velo_decode_kernel(const unsigned long long *__restrict__ key, long n, float *__restrict__ depth)
{
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
		const unsigned long long k = key[p];
		depth[p] = k == NO_POINT ? 0.f : __uint_as_float((unsigned)(k >> 32));
	}
}

long grid_for(long n) { return std::min<long>((n + THREADS - 1) / THREADS, (long)adc_num_sms() * 8); }

// the checks every entry shares: sizes, H * W < 2^31, f and fB > 0, finite cx, cy, doffs, max_depth > 0 (+inf: no cap)
int check_cam(int H, int W, float f, float cx, float cy, float fB, float doffs, float max_depth, Cam *c)
{
	if (H < 1 || W < 1) return ADCENSUS_EINVAL;
	if ((long)H * W >= (1l << 31)) return ADCENSUS_ELIMIT;
	if (!(f > 0.f && fB > 0.f && isfinite(f) && isfinite(fB) && isfinite(cx) && isfinite(cy) && isfinite(doffs) && max_depth > 0.f))
		return ADCENSUS_EINVAL;
	*c = Cam{f, cx, cy, fB, doffs, max_depth};
	return 0;
}

}  // namespace

extern "C" {

int mccnn_disp_to_depth(const float *disp, int H, int W, float f, float cx, float cy, float fB, float doffs, float max_depth,
			float *Z, float *X, float *Y, adcensus_stream_t stream)
{
	Cam c;
	if (!disp || !Z || !X != !Y) return ADCENSUS_EINVAL;
	const int rc = check_cam(H, W, f, cx, cy, fB, doffs, max_depth, &c);
	if (rc) return rc;
	const long n = (long)H * W;
	cudaStream_t s = adc_stream(stream);
	depth_kernel<<<grid_for(n), THREADS, 0, s>>>(disp, n, W, c, Z, X, Y);
	ADC_CHECK_LAUNCH();
	return 0;
}

int mccnn_point_cloud_count(const float *disp, int H, int W, float fB, float doffs, float max_depth, long long *count,
			    adcensus_stream_t stream)
{
	Cam c;
	if (!disp || !count) return ADCENSUS_EINVAL;
	int rc = check_cam(H, W, 1.f, 0.f, 0.f, fB, doffs, max_depth, &c);
	if (rc) return rc;
	const long n = (long)H * W;
	cudaStream_t s = adc_stream(stream);
	int *blk = nullptr;
	rc = adc_scratch_alloc((void **)&blk, sizeof(int) * adc_div_up(n, CHUNK), s);
	if (rc) return rc;
	rc = cloud_scan(disp, n, c, blk, nullptr, count, s);
	const int rf = adc_scratch_free(blk, s);
	return rc ? rc : rf;
}

int mccnn_point_cloud_fill(const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy, float fB,
			   float doffs, float max_depth, unsigned char *out, long long cap, adcensus_stream_t stream)
{
	Cam c;
	if (!disp || !rgb || (nch != 1 && nch != 3) || cap < 0 || (cap && !out) || ((uintptr_t)out & 15)) return ADCENSUS_EINVAL;
	int rc = check_cam(H, W, f, cx, cy, fB, doffs, max_depth, &c);
	if (rc) return rc;
	if (!cap) return 0;
	const long n = (long)H * W;
	const int nblk = adc_div_up(n, CHUNK);
	cudaStream_t s = adc_stream(stream);
	// block offsets and the total (8-byte aligned first), then the block counts
	char *scratch = nullptr;
	rc = adc_scratch_alloc((void **)&scratch, sizeof(long long) * (nblk + 1) + sizeof(int) * nblk, s);
	if (rc) return rc;
	long long *off = (long long *)scratch;
	int *blk = (int *)(off + nblk + 1);
	rc = cloud_scan(disp, n, c, blk, off, off + nblk, s);
	if (!rc) {
		cloud_fill_kernel<<<nblk, THREADS, 0, s>>>(disp, rgb, nch, n, W, c, off, out, cap);
		rc = (int)cudaPeekAtLastError();
	}
	const int rf = adc_scratch_free(scratch, s);
	return rc ? rc : rf;
}

int mccnn_depth_metrics(const float *pred, int pred_depth, const float *gt, int H, int W, float fB, float doffs, float min_depth,
			float max_depth, long long *counts, double *sums, adcensus_stream_t stream)
{
	Cam c;
	if (!pred || !gt || !counts || !sums || !(min_depth > 0.f) || !(min_depth <= max_depth)) return ADCENSUS_EINVAL;
	int rc = check_cam(H, W, 1.f, 0.f, 0.f, fB, doffs, max_depth, &c);
	if (rc) return rc;
	const long n = (long)H * W;
	const int nblk = adc_div_up(n, CHUNK);
	cudaStream_t s = adc_stream(stream);
	double *part = nullptr;
	rc = adc_scratch_alloc((void **)&part, sizeof(double) * NSUM * nblk, s);
	if (rc) return rc;
	rc = (int)cudaMemsetAsync(counts, 0, sizeof(long long) * MCCNN_DEPTH_NCOUNT, s);
	if (!rc) {
		metrics_kernel<<<nblk, THREADS, 0, s>>>(pred, pred_depth, gt, n, c, min_depth, (unsigned long long *)counts, part);
		metrics_finish_kernel<<<1, THREADS, 0, s>>>(part, nblk, sums);
		rc = (int)cudaPeekAtLastError();
	}
	const int rf = adc_scratch_free(part, s);
	return rc ? rc : rf;
}

int mccnn_velo_depth_map(const float *pts, long long n, const float *P, int H, int W, float min_depth, float *depth,
			 adcensus_stream_t stream)
{
	if ((n && !pts) || ((uintptr_t)pts & 15) || !P || !depth || n < 0 || H < 1 || W < 1 || !(min_depth >= 0.f) ||
	    !isfinite(min_depth))
		return ADCENSUS_EINVAL;
	if ((long)H * W >= (1l << 31) || n >= (1ll << 32)) return ADCENSUS_ELIMIT;
	Proj pr;
	for (int k = 0; k < 12; k++) {
		if (!isfinite(P[k])) return ADCENSUS_EINVAL;
		pr.p[k] = P[k];
	}
	const long npx = (long)H * W;
	cudaStream_t s = adc_stream(stream);
	unsigned long long *key = nullptr;
	int rc = adc_scratch_alloc((void **)&key, sizeof(unsigned long long) * npx, s);
	if (rc) return rc;
	rc = (int)cudaMemsetAsync(key, 0xff, sizeof(unsigned long long) * npx, s);
	if (!rc) {
		if (n) velo_key_kernel<<<grid_for(n), THREADS, 0, s>>>((const float4 *)pts, n, pr, H, W, min_depth, key);
		velo_decode_kernel<<<grid_for(npx), THREADS, 0, s>>>(key, npx, depth);
		rc = (int)cudaPeekAtLastError();
	}
	const int rf = adc_scratch_free(key, s);
	return rc ? rc : rf;
}

}  // extern "C"
