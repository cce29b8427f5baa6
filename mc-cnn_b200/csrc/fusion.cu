// fusion.cu -- the stereo depth of posed frames fused into one world-frame voxel map, for sm_90a (DESIGN §23; an addition
// beyond the reference).
//
// The table is a key-sorted structure of arrays: key, n_pix, n_frames, three float64 sums of the world points and three
// int64 sums of the colour bytes.  mccnn_fusion_add runs one frame:
//
// 1. compact: the pixels with a depth (depth.cu's rule, camera.cuh) and a voxel inside the key range, as (key, pixel index)
//    in row-major order (block counts, a 64-bit scan in block order, then each block ranks its pixels by ballots);
// 2. sort: a stable LSD radix sort of the pairs, eight passes of 8 bits over the 63-bit keys (block histograms, their scan
//    in digit-major order, then a scatter that ranks equal digits within each block in element order);
// 3. reduce: the first element of each run of equal keys sums its run sequentially, so a voxel's partial adds its pixels in
//    row-major order, starting at +0.0;
// 4. merge: each frame voxel finds its rank in the table by binary search, the new ones are counted (the one int64 read
//    back, which sizes the destination), then every table voxel and every new frame voxel is written to its place in the
//    destination array, the table's sums plus the frame's partial where the keys are equal.
//
// The world point is computed from the pixel in step 1 and again in step 3, by the same code, so both see the same bits.
// Nothing is summed with float atomics: every run and every GPU gives the same table.
#include <math.h>

#include "camera.cuh"
#include "keysort.cuh"

namespace {

constexpr int REC = 15;                          // bytes per PLY vertex
constexpr long long KEY_HALF = 1ll << 20;
constexpr double KEY_LO = -1048576.0, KEY_HI = 1048576.0;

// device counters of one add
enum { C_M, C_OUT, C_U, C_NEW, C_SCRATCH, C_N };

// A table of `cap` voxels in one allocation: key, n_pix, n_frames, then the three sum planes and the three colour planes.
struct Tab {
	u64 *key;
	long long *npix, *nfr, *col;   // col: 3 planes of cap
	double *sum;                   // 3 planes of cap
	long long cap;
};

__host__ __device__ inline size_t tab_bytes(long long cap) { return (size_t)cap * (3 * 8 + 3 * 8 + 3 * 8); }

Tab tab_at(void *p, long long cap)
{
	Tab t;
	t.key = (u64 *)p;
	t.npix = (long long *)(t.key + cap);
	t.nfr = t.npix + cap;
	t.sum = (double *)(t.nfr + cap);
	t.col = (long long *)(t.sum + 3 * cap);
	t.cap = cap;
	return t;
}

// the world point of pixel p, or false when it has no depth: w = R (X, Y, Z) + t in float64, each operation rounded once
__device__ __forceinline__ bool world_of(float d, long p, int W, const Cam &c, const Pose &T, double *w)
{
	float z;
	if (!depth_of(d, c, &z)) return false;
	const int y = (int)(p / W), x = (int)(p - (long)y * W);
	to_world(lateral(x, c.cx, z, c.f), lateral(y, c.cy, z, c.f), z, T, w);
	return true;
}

// 1 and the key of world point w, or 2 when an axis's voxel index lies outside [-2^20, 2^20)
__device__ __forceinline__ int key_of(const double *w, double v, u64 *key)
{
	u64 k = 0;
#pragma unroll
	for (int a = 0; a < 3; a++) {
		const double q = floor(__ddiv_rn(w[a], v));
		if (!(q >= KEY_LO && q < KEY_HI)) return 2;
		k = k << 21 | (u64)((long long)q + KEY_HALF);
	}
	*key = k;
	return 1;
}

// 0: no point, 1: a point and its key, 2: a point outside the key range
__device__ __forceinline__ int classify(const float *disp, long p, int W, const Cam &c, const Pose &T, double v, u64 *key)
{
	double w[3];
	if (!world_of(disp[p], p, W, c, T, w)) return 0;
	return key_of(w, v, key);
}

// ---- 1. compaction ----

__global__ void __launch_bounds__(THREADS) compact_count_kernel(const float *__restrict__ disp, long n, int W, Cam c, Pose T, double v,
								int *__restrict__ blk, unsigned long long *__restrict__ outside)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0, o = 0;
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + threadIdx.x;
		u64 key;
		const int r = p < n ? classify(disp, p, W, c, T, v, &key) : 0;
		k += r == 1;
		o += r == 2;
	}
	k = block_sum(k, warp_n);
	o = block_sum(o, warp_n);
	if (threadIdx.x == 0) {
		blk[blockIdx.x] = k;
		if (o) atomicAdd(outside, (unsigned long long)o);
	}
}

__global__ void __launch_bounds__(THREADS) compact_fill_kernel(const float *__restrict__ disp, long n, int W, Cam c, Pose T, double v,
							       const long long *__restrict__ off, u64 *__restrict__ keys,
							       int *__restrict__ vals)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	long long at = off[blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		const long p = base + (long)i * THREADS + threadIdx.x;
		u64 key = 0;
		const bool ok = p < n && classify(disp, p, W, c, T, v, &key) == 1;
		int all;
		const int r = round_rank(ok, warp_n, &all);
		if (ok) {
			keys[at + r] = key;
			vals[at + r] = (int)p;
		}
		at += all;
	}
}

// ---- 3. one partial per run of equal keys ----

__device__ __forceinline__ bool is_head(const u64 *keys, long i, long long n) { return i < n && (i == 0 || keys[i] != keys[i - 1]); }

__global__ void __launch_bounds__(THREADS) head_count_kernel(const u64 *__restrict__ keys, const long long *__restrict__ dn,
							     int *__restrict__ blk)
{
	__shared__ int warp_n[THREADS / 32];
	const long long n = *dn;
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0;
	for (int i = 0; i < ITEMS; i++) k += is_head(keys, base + (long)i * THREADS + threadIdx.x, n);
	k = block_sum(k, warp_n);
	if (threadIdx.x == 0) blk[blockIdx.x] = k;
}

__global__ void __launch_bounds__(THREADS) reduce_kernel(const u64 *__restrict__ keys, const int *__restrict__ vals,
							 const long long *__restrict__ dn, const long long *__restrict__ off,
							 const float *__restrict__ disp, const unsigned char *__restrict__ rgb, int nch,
							 int W, Cam c, Pose T, Tab frm)
{
	__shared__ int warp_n[THREADS / 32];
	const long long n = *dn;
	const long base = (long)blockIdx.x * CHUNK;
	long long at = off[blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		const bool head = is_head(keys, e, n);
		int all;
		const int r = round_rank(head, warp_n, &all);
		if (head) {
			const u64 k = keys[e];
			double s[3] = {0.0, 0.0, 0.0};
			long long col[3] = {0, 0, 0}, np = 0;
			for (long j = e; j < n && keys[j] == k; j++, np++) {
				const int p = vals[j];
				double w[3];
				world_of(disp[p], p, W, c, T, w);
#pragma unroll
				for (int a = 0; a < 3; a++) {
					s[a] = __dadd_rn(s[a], w[a]);
					col[a] += rgb[nch == 3 ? 3l * p + a : (long)p];
				}
			}
			const long long u = at + r;
			frm.key[u] = k;
			frm.npix[u] = np;
#pragma unroll
			for (int a = 0; a < 3; a++) {
				frm.sum[a * frm.cap + u] = s[a];
				frm.col[a * frm.cap + u] = col[a];
			}
		}
		at += all;
	}
}

// ---- 4. merge into the table ----

// table voxel i goes to i + (new frame voxels below its key), with the frame's partial added when the frame has its key
__global__ void merge_table_kernel(Tab src, long long n, Tab frm, const long long *__restrict__ dU, const long long *__restrict__ nn,
				   const long long *__restrict__ dnew, Tab dst)
{
	const long long U = *dU, nnew = *dnew;
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		const u64 k = src.key[i];
		const long long ub = lower_bound(frm.key, U, k);
		const long long pos = i + (ub < U ? nn[ub] : nnew);
		const bool both = ub < U && frm.key[ub] == k;
		dst.key[pos] = k;
		dst.npix[pos] = src.npix[i] + (both ? frm.npix[ub] : 0);
		dst.nfr[pos] = src.nfr[i] + both;
#pragma unroll
		for (int a = 0; a < 3; a++) {
			const double s = src.sum[a * src.cap + i];
			dst.sum[a * dst.cap + pos] = both ? __dadd_rn(s, frm.sum[a * frm.cap + ub]) : s;
			dst.col[a * dst.cap + pos] = src.col[a * src.cap + i] + (both ? frm.col[a * frm.cap + ub] : 0);
		}
	}
}

// a frame voxel absent from the table goes to (table voxels below its key) + (new frame voxels before it)
__global__ void merge_frame_kernel(Tab frm, const long long *__restrict__ dU, const long long *__restrict__ lb,
				   const long long *__restrict__ nn, const u64 *__restrict__ tkey, long long n, Tab dst)
{
	const long long U = *dU;
	for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < U; j += (long long)gridDim.x * blockDim.x) {
		const u64 k = frm.key[j];
		const long long l = lb[j];
		if (!fresh(tkey, n, l, k)) continue;
		const long long pos = l + nn[j];
		dst.key[pos] = k;
		dst.npix[pos] = frm.npix[j];
		dst.nfr[pos] = 1;
#pragma unroll
		for (int a = 0; a < 3; a++) {
			dst.sum[a * dst.cap + pos] = __dadd_rn(0.0, frm.sum[a * frm.cap + j]);
			dst.col[a * dst.cap + pos] = frm.col[a * frm.cap + j];
		}
	}
}

__global__ void stats_kernel(const unsigned long long *__restrict__ ctr, long long n, long long *__restrict__ stats)
{
	stats[0] = (long long)ctr[C_M];
	stats[1] = (long long)ctr[C_OUT];
	stats[2] = n;
}

// ---- output ----

__global__ void __launch_bounds__(THREADS) out_count_kernel(const long long *__restrict__ nfr, long long n, int min_frames,
							    int *__restrict__ blk)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0;
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		k += e < n && nfr[e] >= min_frames;
	}
	k = block_sum(k, warp_n);
	if (threadIdx.x == 0) blk[blockIdx.x] = k;
}

__device__ __forceinline__ void put_float(unsigned char *p, float v)
{
	const unsigned u = __float_as_uint(v);
	p[0] = (unsigned char)u;
	p[1] = (unsigned char)(u >> 8);
	p[2] = (unsigned char)(u >> 16);
	p[3] = (unsigned char)(u >> 24);
}

__global__ void __launch_bounds__(THREADS) out_fill_kernel(Tab t, long long n, int min_frames, const long long *__restrict__ off,
							   unsigned char *__restrict__ out, long long cap)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	long long at = off[blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		const bool ok = e < n && t.nfr[e] >= min_frames;
		int all;
		const int r = round_rank(ok, warp_n, &all);
		if (ok && at + r < cap) {
			unsigned char *rec = out + REC * (at + r);
			const long long np = t.npix[e];
			for (int a = 0; a < 3; a++) {
				put_float(rec + 4 * a, __double2float_rn(__ddiv_rn(t.sum[a * t.cap + e], (double)np)));
				rec[12 + a] = (unsigned char)((t.col[a * t.cap + e] + np / 2) / np);
			}
		}
		at += all;
	}
}

}  // namespace

struct mccnn_fusion {
	double voxel;
	int device;
	long long n;                 // voxels in the table
	int cur;                     // tab[cur] holds the table, tab[1 - cur] receives the next merge
	void *mem[2];
	Tab tab[2];
	// per-frame scratch, sized for `px` pixels
	long px;
	void *scratch;
	u64 *keyA, *keyB;
	int *valA, *valB, *blk, *hist;
	long long *off, *hoff, *lb, *nn;
	unsigned long long *ctr;
	Tab frm;
};

namespace {

int grow_scratch(mccnn_fusion *h, long px)
{
	if (px <= h->px) return 0;
	const long nblk = adc_div_up(px, CHUNK);
	const size_t bytes = 2 * 8 * (size_t)px + 2 * 4 * (size_t)px + 4 * (size_t)nblk + 4 * (size_t)BINS * nblk +
			     8 * (size_t)(nblk + 1) + 8 * (size_t)(BINS * nblk + 1) + 2 * 8 * (size_t)px + 8 * C_N + tab_bytes(px) + 64;
	if (h->scratch) ADC_CUDA(cudaFree(h->scratch));
	h->scratch = nullptr;
	h->px = 0;
	ADC_CUDA(cudaMalloc(&h->scratch, bytes));
	char *p = (char *)h->scratch;
	auto take = [&p](size_t b) {
		char *q = p;
		p += (b + 7) & ~(size_t)7;
		return q;
	};
	h->frm = tab_at(take(tab_bytes(px)), px);
	h->keyA = (u64 *)take(8 * (size_t)px);
	h->keyB = (u64 *)take(8 * (size_t)px);
	h->lb = (long long *)take(8 * (size_t)px);
	h->nn = (long long *)take(8 * (size_t)px);
	h->off = (long long *)take(8 * (size_t)(nblk + 1));
	h->hoff = (long long *)take(8 * (size_t)(BINS * nblk + 1));
	h->ctr = (unsigned long long *)take(8 * C_N);
	h->valA = (int *)take(4 * (size_t)px);
	h->valB = (int *)take(4 * (size_t)px);
	h->blk = (int *)take(4 * (size_t)nblk);
	h->hist = (int *)take(4 * (size_t)BINS * nblk);
	h->px = px;
	return 0;
}

// makes tab[slot] hold at least `need` voxels; its contents are not kept
int reserve(mccnn_fusion *h, int slot, long long need)
{
	if (h->mem[slot] && h->tab[slot].cap >= need) return 0;
	const long long cap = std::max<long long>(need + need / 2, 4096);
	if (h->mem[slot]) ADC_CUDA(cudaFree(h->mem[slot]));
	h->mem[slot] = nullptr;
	ADC_CUDA(cudaMalloc(&h->mem[slot], tab_bytes(cap)));
	h->tab[slot] = tab_at(h->mem[slot], cap);
	return 0;
}

int run_add(mccnn_fusion *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, const Cam &c, const Pose &T,
	    long long *stats, cudaStream_t s)
{
	const long n = (long)H * W;
	const int nblk = adc_div_up(n, CHUNK);
	int rc = grow_scratch(h, n);
	if (rc) return rc;
	ADC_CUDA(cudaMemsetAsync(h->ctr, 0, 8 * C_N, s));
	long long *ctr = (long long *)h->ctr;
	// 1. compaction
	compact_count_kernel<<<nblk, THREADS, 0, s>>>(disp, n, W, c, T, h->voxel, h->blk, h->ctr + C_OUT);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_M);
	compact_fill_kernel<<<nblk, THREADS, 0, s>>>(disp, n, W, c, T, h->voxel, h->off, h->keyA, h->valA);
	ADC_CHECK_LAUNCH();
	// 2. sort: eight passes end where they started, in keyA / valA
	radix_sort_pairs(h->keyA, h->valA, h->keyB, h->valB, ctr + C_M, nblk, h->hist, h->hoff, ctr + C_SCRATCH, s);
	ADC_CHECK_LAUNCH();
	// 3. one partial per voxel
	head_count_kernel<<<nblk, THREADS, 0, s>>>(h->keyA, ctr + C_M, h->blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_U);
	reduce_kernel<<<nblk, THREADS, 0, s>>>(h->keyA, h->valA, ctr + C_M, h->off, disp, rgb, nch, W, c, T, h->frm);
	// 4. merge
	const Tab &src = h->tab[h->cur];
	const long long tn = h->n;
	const u64 *tkey = h->mem[h->cur] ? src.key : nullptr;
	match_count_kernel<<<nblk, THREADS, 0, s>>>(h->frm.key, ctr + C_U, tkey, tn, h->lb, h->blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_NEW);
	match_rank_kernel<<<nblk, THREADS, 0, s>>>(h->frm.key, ctr + C_U, tkey, tn, h->lb, h->off, h->nn);
	ADC_CHECK_LAUNCH();
	long long nnew = 0;
	ADC_CUDA(cudaMemcpyAsync(&nnew, ctr + C_NEW, sizeof nnew, cudaMemcpyDeviceToHost, s));
	ADC_CUDA(cudaStreamSynchronize(s));
	const int dst = 1 - h->cur;
	rc = reserve(h, dst, tn + nnew);
	if (rc) return rc;
	if (tn) merge_table_kernel<<<grid_for(tn), THREADS, 0, s>>>(src, tn, h->frm, ctr + C_U, h->nn, ctr + C_NEW, h->tab[dst]);
	merge_frame_kernel<<<grid_for(n), THREADS, 0, s>>>(h->frm, ctr + C_U, h->lb, h->nn, tkey, tn, h->tab[dst]);
	stats_kernel<<<1, 1, 0, s>>>(h->ctr, tn + nnew, stats);
	ADC_CHECK_LAUNCH();
	h->cur = dst;
	h->n = tn + nnew;
	return 0;
}

}  // namespace

extern "C" {

int mccnn_fusion_create(mccnn_fusion **out, double voxel, int device)
{
	if (!out) return ADCENSUS_EINVAL;
	*out = nullptr;
	int ndev = 0;
	if (!(voxel > 0.0) || !isfinite(voxel)) return ADCENSUS_EINVAL;
	ADC_CUDA(cudaGetDeviceCount(&ndev));
	if (device < 0 || device >= ndev) return ADCENSUS_EINVAL;
	mccnn_fusion *h = new mccnn_fusion();
	h->voxel = voxel;
	h->device = device;
	*out = h;
	return 0;
}

int mccnn_fusion_add(mccnn_fusion *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy,
		     float fB, float doffs, float max_depth, const double *pose12, long long *stats, adcensus_stream_t stream)
{
	if (!h || !disp || !rgb || !stats || (nch != 1 && nch != 3) || H < 1 || W < 1) return ADCENSUS_EINVAL;
	if ((long)H * W * nch >= (1l << 31)) return ADCENSUS_ELIMIT;
	if (!(f > 0.f && fB > 0.f && isfinite(f) && isfinite(fB) && isfinite(cx) && isfinite(cy) && isfinite(doffs) && max_depth > 0.f))
		return ADCENSUS_EINVAL;
	Pose T;
	int rc = check_pose(pose12, &T);
	if (rc) return rc;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	return run_add(h, disp, rgb, nch, H, W, Cam{f, cx, cy, fB, doffs, max_depth}, T, stats, adc_stream(stream));
}

long long mccnn_fusion_size(const mccnn_fusion *h) { return h ? h->n : -1; }

int mccnn_fusion_count(const mccnn_fusion *h, int min_frames, long long *count, adcensus_stream_t stream)
{
	if (!h || !count || min_frames < 1) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	const long long n = h->n;
	if (!n) return (int)cudaMemsetAsync(count, 0, sizeof(long long), s);
	const long long nblk = (n + CHUNK - 1) / CHUNK;
	int *blk = nullptr;
	int rc = adc_scratch_alloc((void **)&blk, sizeof(int) * nblk + sizeof(long long) * nblk + 8, s);
	if (rc) return rc;
	long long *off = (long long *)((char *)blk + ((sizeof(int) * nblk + 7) & ~(size_t)7));
	out_count_kernel<<<(unsigned)nblk, THREADS, 0, s>>>(h->tab[h->cur].nfr, n, min_frames, blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(blk, nblk, off, count);
	rc = (int)cudaPeekAtLastError();
	const int rf = adc_scratch_free(blk, s);
	return rc ? rc : rf;
}

int mccnn_fusion_fill(const mccnn_fusion *h, int min_frames, unsigned char *out, long long cap, adcensus_stream_t stream)
{
	if (!h || min_frames < 1 || cap < 0 || (cap && !out)) return ADCENSUS_EINVAL;
	const long long n = h->n;
	if (!cap || !n) return 0;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	const long long nblk = (n + CHUNK - 1) / CHUNK;
	int *blk = nullptr;
	int rc = adc_scratch_alloc((void **)&blk, sizeof(int) * nblk + sizeof(long long) * (nblk + 1) + 8, s);
	if (rc) return rc;
	long long *off = (long long *)((char *)blk + ((sizeof(int) * nblk + 7) & ~(size_t)7));
	out_count_kernel<<<(unsigned)nblk, THREADS, 0, s>>>(h->tab[h->cur].nfr, n, min_frames, blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(blk, nblk, off, off + nblk);
	out_fill_kernel<<<(unsigned)nblk, THREADS, 0, s>>>(h->tab[h->cur], n, min_frames, off, out, cap);
	rc = (int)cudaPeekAtLastError();
	const int rf = adc_scratch_free(blk, s);
	return rc ? rc : rf;
}

int mccnn_fusion_table(const mccnn_fusion *h, unsigned long long *keys, long long *npix, long long *nframes, double *sums,
		       long long *colours, adcensus_stream_t stream)
{
	if (!h) return ADCENSUS_EINVAL;
	const long long n = h->n;
	if (!n) return 0;
	if (!keys || !npix || !nframes || !sums || !colours) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	const Tab &t = h->tab[h->cur];
	ADC_CUDA(cudaMemcpyAsync(keys, t.key, 8 * n, cudaMemcpyDeviceToDevice, s));
	ADC_CUDA(cudaMemcpyAsync(npix, t.npix, 8 * n, cudaMemcpyDeviceToDevice, s));
	ADC_CUDA(cudaMemcpyAsync(nframes, t.nfr, 8 * n, cudaMemcpyDeviceToDevice, s));
	for (int a = 0; a < 3; a++) {
		ADC_CUDA(cudaMemcpyAsync(sums + a * n, t.sum + a * t.cap, 8 * n, cudaMemcpyDeviceToDevice, s));
		ADC_CUDA(cudaMemcpyAsync(colours + a * n, t.col + a * t.cap, 8 * n, cudaMemcpyDeviceToDevice, s));
	}
	return 0;
}

void mccnn_fusion_destroy(mccnn_fusion *h)
{
	if (!h) return;
	{
		DeviceScope dev(h->device);
		if (!dev.rc) {
			for (void *p : {h->mem[0], h->mem[1], h->scratch})
				if (p) cudaFree(p);
		}
	}
	delete h;
}

}  // extern "C"
