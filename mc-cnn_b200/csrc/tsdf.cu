// tsdf.cu -- the stereo depth of posed frames fused into a truncated signed distance field, for sm_90a (DESIGN §24; an
// addition beyond the reference).
//
// The field is a table of bricks of 8^3 voxels: a key-sorted array of (brick key, slot) pairs, the slot pointing into an
// append-only pool of bricks.  A brick holds, per voxel, S (float64), n, nc and three colour sums (int32), as planes of
// 512 in the local order (z, y, x): 28 bytes per voxel, 14336 per brick.  mccnn_tsdf_add runs one frame:
//
// 1. allocate: each valid pixel's 2K + 1 ray points around its depth, as brick keys (block counts, a 64-bit scan in block
//    order, ballot ranks), sorted by keysort.cuh's radix sort, one key per run; each finds its rank in the table by binary
//    search, the new ones are counted (the one int64 read back), and the (key, slot) pairs are merged into the other half
//    of the double-buffered key array, the new bricks taking the next pool slots, zeroed;
// 2. integrate: one thread per voxel of every brick of the table projects the voxel centre into the frame and updates
//    the voxel at most once.
//
// mccnn_tsdf_mesh_* extract marching tetrahedra on the Kuhn split (vertex counts, a scan, vertices, then faces) and
// mccnn_tsdf_render casts rays through the field.  Nothing is summed with atomics: every run and every GPU gives the same
// field, mesh and maps.
#include <math.h>

#include "camera.cuh"
#include "keysort.cuh"

namespace {

constexpr int REC = 15;                          // bytes per PLY vertex
constexpr int VOX = 512;                         // voxels per brick, one thread each
constexpr long long BRICK_BYTES = VOX * 28;      // S, n, nc, 3 colour planes
constexpr long long KEY_HALF = 1ll << 20;
constexpr double KEY_LO = -1048576.0, KEY_HI = 1048576.0;
constexpr int MAX_FRAMES = 1 << 23;              // 255 2^23 + 2^22 < 2^31: the int32 colour sums cannot overflow
constexpr u64 EMPTY = ~0ull;                     // no key: keys are below 2^63

// device counters of one add: allocation points, outside points, valid pixels, unique keys, new keys, scratch
enum { C_M, C_OUT, C_PIX, C_U, C_NEW, C_SCRATCH, C_N };

// the edge directions x, y, z, xy, xz, yz, xyz as corner bits (x 1, y 2, z 4), in vertex order
__constant__ int DIR_BITS[7] = {1, 2, 4, 3, 5, 6, 7};
// the direction index of corner bits 1 .. 7
__constant__ int DIR_OF[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
// the Kuhn tetrahedra {0, e_p1, e_p1 + e_p2, 7} over the axis permutations (x y z, x z y, y x z, y z x, z x y, z y x) and
// the permutation's parity: an odd one is negatively oriented
__constant__ int TET[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ int TET_ODD[6] = {0, 1, 1, 0, 0, 1};
// even reorderings of a tetrahedron's corners: the lone corner first, and the two negative corners first
__constant__ int ORD1[4][4] = {{0, 1, 2, 3}, {1, 0, 3, 2}, {2, 3, 0, 1}, {3, 2, 1, 0}};
__constant__ int ORD2[4][4][4] = {{{0}, {0, 1, 2, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}},
				  {{0}, {0}, {1, 2, 0, 3}, {1, 3, 2, 0}},
				  {{0}, {0}, {0}, {2, 3, 0, 1}}};

__device__ __forceinline__ double *b_S(char *pool, long long s) { return (double *)(pool + s * BRICK_BYTES); }
__device__ __forceinline__ int *b_n(char *pool, long long s) { return (int *)(pool + s * BRICK_BYTES + 8 * VOX); }
__device__ __forceinline__ int *b_nc(char *pool, long long s) { return (int *)(pool + s * BRICK_BYTES + 12 * VOX); }
__device__ __forceinline__ int *b_col(char *pool, long long s, int a) { return (int *)(pool + s * BRICK_BYTES + (16 + 4 * a) * VOX); }

__device__ __forceinline__ void brick_of_key(u64 k, long long *b)
{
	b[0] = (long long)(k >> 42) - KEY_HALF;
	b[1] = (long long)((k >> 21) & ((1ull << 21) - 1)) - KEY_HALF;
	b[2] = (long long)(k & ((1ull << 21) - 1)) - KEY_HALF;
}

// the key of brick b, or false when an axis lies outside [-2^20, 2^20)
__device__ __forceinline__ bool key_of_brick(const long long *b, u64 *key)
{
	u64 k = 0;
	for (int a = 0; a < 3; a++) {
		if (b[a] < -KEY_HALF || b[a] >= KEY_HALF) return false;
		k = k << 21 | (u64)(b[a] + KEY_HALF);
	}
	*key = k;
	return true;
}

// ---- 1. allocation ----

// element e = p (2K + 1) + j + K: 0 no point, 1 a point and its brick key, 2 a point whose brick lies outside the key range;
// *pix: the pixel has a depth (set for j = 0)
__device__ __forceinline__ int classify(const float *disp, long e, int J, int W, const Cam &c, const Pose &T, float step, double v,
					 u64 *key, bool *pix)
{
	const long p = e / J;
	const int j = (int)(e - p * J) - J / 2;
	float Z;
	*pix = false;
	if (!depth_of(disp[p], c, &Z)) return 0;
	*pix = j == 0;
	const float z = __fadd_rn(Z, __fmul_rn((float)j, step));
	if (!(z > 0.f)) return 0;
	const int y = (int)(p / W), x = (int)(p - (long)y * W);
	double w[3];
	to_world(lateral(x, c.cx, z, c.f), lateral(y, c.cy, z, c.f), z, T, w);
	u64 k = 0;
#pragma unroll
	for (int a = 0; a < 3; a++) {
		const double b = floor(__dmul_rn(floor(__ddiv_rn(w[a], v)), 0.125));
		if (!(b >= KEY_LO && b < KEY_HI)) return 2;
		k = k << 21 | (u64)((long long)b + KEY_HALF);
	}
	*key = k;
	return 1;
}

__global__ void __launch_bounds__(THREADS) alloc_count_kernel(const float *__restrict__ disp, long m, int J, int W, Cam c, Pose T,
							      float step, double v, int *__restrict__ blk,
							      unsigned long long *__restrict__ ctr)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	int k = 0, o = 0, px = 0;
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		u64 key;
		bool pix = false;
		const int r = e < m ? classify(disp, e, J, W, c, T, step, v, &key, &pix) : 0;
		k += r == 1;
		o += r == 2;
		px += pix;
	}
	k = block_sum(k, warp_n);
	o = block_sum(o, warp_n);
	px = block_sum(px, warp_n);
	if (threadIdx.x == 0) {
		blk[blockIdx.x] = k;
		if (o) atomicAdd(ctr + C_OUT, (unsigned long long)o);
		if (px) atomicAdd(ctr + C_PIX, (unsigned long long)px);
	}
}

__global__ void __launch_bounds__(THREADS) alloc_fill_kernel(const float *__restrict__ disp, long m, int J, int W, Cam c, Pose T,
							     float step, double v, const long long *__restrict__ off,
							     u64 *__restrict__ keys, int *__restrict__ vals)
{
	__shared__ int warp_n[THREADS / 32];
	const long base = (long)blockIdx.x * CHUNK;
	long long at = off[blockIdx.x];
	for (int i = 0; i < ITEMS; i++) {
		const long e = base + (long)i * THREADS + threadIdx.x;
		u64 key = 0;
		bool pix;
		const bool ok = e < m && classify(disp, e, J, W, c, T, step, v, &key, &pix) == 1;
		int all;
		const int r = round_rank(ok, warp_n, &all);
		if (ok) {
			keys[at + r] = key;
			vals[at + r] = (int)(e / J);
		}
		at += all;
	}
}

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

__global__ void __launch_bounds__(THREADS) head_fill_kernel(const u64 *__restrict__ keys, const long long *__restrict__ dn,
							    const long long *__restrict__ off, u64 *__restrict__ uniq)
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
		if (head) uniq[at + r] = keys[e];
		at += all;
	}
}

// table brick i keeps its slot and goes to i + (new frame bricks below its key)
__global__ void merge_table_kernel(const u64 *__restrict__ skey, const long long *__restrict__ sslot, long long n,
				   const u64 *__restrict__ fkey, const long long *__restrict__ dU, const long long *__restrict__ nn,
				   const long long *__restrict__ dnew, u64 *__restrict__ dkey, long long *__restrict__ dslot)
{
	const long long U = *dU, nnew = *dnew;
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		const u64 k = skey[i];
		const long long ub = lower_bound(fkey, U, k);
		const long long pos = i + (ub < U ? nn[ub] : nnew);
		dkey[pos] = k;
		dslot[pos] = sslot[i];
	}
}

// a new frame brick goes to (table bricks below its key) + (new frame bricks before it) and takes pool slot n + the latter;
// the brick-index bounds grow to hold it
__global__ void merge_frame_kernel(const u64 *__restrict__ fkey, const long long *__restrict__ dU, const long long *__restrict__ lb,
				   const long long *__restrict__ nn, const u64 *__restrict__ tkey, long long n, u64 *__restrict__ dkey,
				   long long *__restrict__ dslot, long long *__restrict__ box)
{
	const long long U = *dU;
	for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < U; j += (long long)gridDim.x * blockDim.x) {
		const u64 k = fkey[j];
		const long long l = lb[j];
		if (!fresh(tkey, n, l, k)) continue;
		dkey[l + nn[j]] = k;
		dslot[l + nn[j]] = n + nn[j];
		long long b[3];
		brick_of_key(k, b);
		for (int a = 0; a < 3; a++) {
			atomicMin(box + a, b[a]);
			atomicMax(box + 3 + a, b[a]);
		}
	}
}

// ---- 2. integration ----

struct Proj {
	int H, W;
	double f, cx, cy;
};

// the pixel index voxel centre c projects to, or -1: q = R^T (c - t) in float64, each operation rounded once; q_z > 0; the
// nearest pixel floor(q_x / q_z f + c_x + 0.5) (likewise y) inside the image
__device__ __forceinline__ long project(const double *c, const Pose &T, const Proj &P, double *qz)
{
	double d[3], q[3];
	for (int a = 0; a < 3; a++) d[a] = __dsub_rn(c[a], T.r[4 * a + 3]);
	for (int a = 0; a < 3; a++) q[a] = __dadd_rn(__dadd_rn(__dmul_rn(T.r[a], d[0]), __dmul_rn(T.r[4 + a], d[1])), __dmul_rn(T.r[8 + a], d[2]));
	*qz = q[2];
	if (!(q[2] > 0.0)) return -1;
	const double u = floor(__dadd_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[0], q[2]), P.f), P.cx), 0.5));
	const double w = floor(__dadd_rn(__dadd_rn(__dmul_rn(__ddiv_rn(q[1], q[2]), P.f), P.cy), 0.5));
	if (!(u >= 0.0 && u < P.W && w >= 0.0 && w < P.H)) return -1;
	return (long)w * P.W + (long)u;
}

__device__ __forceinline__ void voxel_centre(const long long *b, int l, double v, double *c)
{
	const int lx = l & 7, ly = (l >> 3) & 7, lz = l >> 6;
	const int ll[3] = {lx, ly, lz};
	for (int a = 0; a < 3; a++) c[a] = __dmul_rn((double)(8 * b[a] + ll[a]) + 0.5, v);
}

__global__ void __launch_bounds__(VOX) integrate_kernel(const u64 *__restrict__ key, const long long *__restrict__ slot, char *pool,
							const float *__restrict__ disp, const unsigned char *__restrict__ rgb, int nch, Cam c,
							Proj P, Pose T, double v, double mu)
{
	const long long i = blockIdx.x;
	const int l = threadIdx.x;
	long long b[3];
	brick_of_key(key[i], b);
	double ctr[3], qz;
	voxel_centre(b, l, v, ctr);
	const long p = project(ctr, T, P, &qz);
	if (p < 0) return;
	float Z;
	if (!depth_of(disp[p], c, &Z)) return;
	const double eta = __dsub_rn((double)Z, qz);
	if (eta < -mu) return;
	const long long s = slot[i];
	b_S(pool, s)[l] = __dadd_rn(b_S(pool, s)[l], __ddiv_rn(fmin(eta, mu), mu));
	b_n(pool, s)[l] += 1;
	if (fabs(eta) < mu) {
		for (int a = 0; a < 3; a++) b_col(pool, s, a)[l] += rgb[nch == 3 ? 3l * p + a : (long)p];
		b_nc(pool, s)[l] += 1;
	}
}

// ---- reading the field ----

struct Field {
	const u64 *key;
	const long long *slot;
	long long n;
	char *pool;
	double v;
	int min_frames;
};

// phi = S / n of voxel l of the brick in pool slot s, false when the slot is absent or the voxel not observed
__device__ __forceinline__ bool phi_at(const Field &F, long long s, int l, double *phi)
{
	if (s < 0) return false;
	const int n = b_n(F.pool, s)[l];
	if (n < F.min_frames) return false;
	*phi = __ddiv_rn(b_S(F.pool, s)[l], (double)n);
	return true;
}

// the table index of the brick at b + (corner bits o), or -1
__device__ __forceinline__ long long neighbour(const Field &F, const long long *b, int o)
{
	const long long nb[3] = {b[0] + (o & 1), b[1] + ((o >> 1) & 1), b[2] + ((o >> 2) & 1)};
	u64 k;
	if (!key_of_brick(nb, &k)) return -1;
	const long long at = lower_bound(F.key, F.n, k);
	return at < F.n && F.key[at] == k ? at : -1;
}

// an exclusive scan of one value per thread over a block of VOX threads, in thread order; *total the block's sum
__device__ __forceinline__ int block_scan(int x, int *warp_s, int *total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	int inc = x;
	for (int d = 1; d < 32; d <<= 1) {
		const int y = __shfl_up_sync(FULL, inc, d);
		if (lane >= d) inc += y;
	}
	if (lane == 31) warp_s[warp] = inc;
	__syncthreads();
	int before = 0, t = 0;
	for (int w = 0; w < VOX / 32; w++) {
		before += w < warp ? warp_s[w] : 0;
		t += warp_s[w];
	}
	__syncthreads();
	*total = t;
	return before + inc - x;
}

// the block's neighbour table indices (corner bits 0 .. 7, 0 the brick itself) and their pool slots
__device__ __forceinline__ void load_neighbours(const Field &F, long long i, const long long *b, long long *nidx, long long *nslot)
{
	if (threadIdx.x < 8) {
		const long long at = threadIdx.x == 0 ? i : neighbour(F, b, threadIdx.x);
		nidx[threadIdx.x] = at;
		nslot[threadIdx.x] = at < 0 ? -1 : F.slot[at];
	}
	__syncthreads();
}

// corner bits o of the cube whose lower corner is local voxel l: (which neighbour, local voxel)
__device__ __forceinline__ int corner(int l, int o, int *local)
{
	const int x = (l & 7) + (o & 1), y = ((l >> 3) & 7) + ((o >> 1) & 1), z = (l >> 6) + ((o >> 2) & 1);
	*local = ((z & 7) << 6) | ((y & 7) << 3) | (x & 7);
	return (x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2);
}

// the 8 corners of the cube at local voxel l: observed flags (bit per corner) and phi
__device__ __forceinline__ int cube(const Field &F, const long long *nslot, int l, double *phi)
{
	int obs = 0;
	for (int o = 0; o < 8; o++) {
		int lo;
		const int nb = corner(l, o, &lo);
		if (phi_at(F, nslot[nb], lo, phi + o)) obs |= 1 << o;
	}
	return obs;
}

__device__ __forceinline__ int edge_mask(int obs, const double *phi)
{
	int m = 0;
	if (!(obs & 1)) return 0;
	for (int d = 0; d < 7; d++) {
		const int o = DIR_BITS[d];
		if ((obs >> o & 1) && ((phi[0] < 0.0) != (phi[o] < 0.0))) m |= 1 << d;
	}
	return m;
}

__device__ __forceinline__ int tri_count(int obs, const double *phi, int t)
{
	int neg = 0;
	for (int k = 0; k < 4; k++) {
		if (!(obs >> TET[t][k] & 1)) return 0;
		neg += phi[TET[t][k]] < 0.0;
	}
	return neg == 2 ? 2 : (neg & 1);
}

__device__ __forceinline__ int face_count(int obs, const double *phi)
{
	int f = 0;
	for (int t = 0; t < 6; t++) f += tri_count(obs, phi, t);
	return f;
}

// per brick: the edge mask of each voxel, and the brick's vertex and face counts
__global__ void __launch_bounds__(VOX) mesh_count_kernel(Field F, unsigned char *__restrict__ mask, int *__restrict__ vb,
							 int *__restrict__ fb)
{
	__shared__ long long nidx[8], nslot[8];
	__shared__ int warp_s[VOX / 32];
	const long long i = blockIdx.x;
	const int l = threadIdx.x;
	long long b[3];
	brick_of_key(F.key[i], b);
	load_neighbours(F, i, b, nidx, nslot);
	double phi[8];
	const int obs = cube(F, nslot, l, phi);
	const int m = edge_mask(obs, phi);
	mask[i * VOX + l] = (unsigned char)m;
	int tv, tf;
	block_scan(__popc(m), warp_s, &tv);
	block_scan(face_count(obs, phi), warp_s, &tf);
	if (l == 0) {
		vb[i] = tv;
		fb[i] = tf;
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

// per brick: each voxel's first vertex index, and its vertices in direction order
__global__ void __launch_bounds__(VOX) mesh_vertex_kernel(Field F, const unsigned char *__restrict__ mask, const long long *__restrict__ voff,
							  long long *__restrict__ vbase, unsigned char *__restrict__ out, long long cap)
{
	__shared__ long long nidx[8], nslot[8];
	__shared__ int warp_s[VOX / 32];
	const long long i = blockIdx.x;
	const int l = threadIdx.x;
	long long b[3];
	brick_of_key(F.key[i], b);
	load_neighbours(F, i, b, nidx, nslot);
	const int m = mask[i * VOX + l];
	int tv;
	long long at = voff[i] + block_scan(__popc(m), warp_s, &tv);
	vbase[i * VOX + l] = at;
	if (!m) return;
	double phi[8], ca[3], cb[3];
	cube(F, nslot, l, phi);
	voxel_centre(b, l, F.v, ca);
	for (int d = 0; d < 7; d++) {
		if (!(m >> d & 1)) continue;
		const int o = DIR_BITS[d];
		const double t = __ddiv_rn(phi[0], __dsub_rn(phi[0], phi[o]));
		if (at < cap) {
			unsigned char *rec = out + REC * at;
			for (int a = 0; a < 3; a++) {
				cb[a] = __dmul_rn((double)(8 * b[a] + ((l >> (3 * a)) & 7) + ((o >> a) & 1)) + 0.5, F.v);
				put_float(rec + 4 * a, __double2float_rn(__dadd_rn(ca[a], __dmul_rn(t, __dsub_rn(cb[a], ca[a])))));
			}
			// the endpoint nearer the surface, else the other, else none
			int lb;
			const long long sb = nslot[corner(l, o, &lb)], sa = nslot[0];
			const bool near_a = t < 0.5;
			long long s1 = near_a ? sa : sb, s2 = near_a ? sb : sa;
			int l1 = near_a ? l : lb, l2 = near_a ? lb : l;
			if (!b_nc(F.pool, s1)[l1]) {
				s1 = s2;
				l1 = l2;
			}
			const int nc = b_nc(F.pool, s1)[l1];
			for (int a = 0; a < 3; a++) rec[12 + a] = nc ? (unsigned char)((b_col(F.pool, s1, a)[l1] + nc / 2) / nc) : 0;
		}
		at++;
	}
}

// per brick: each voxel's triangles, tetrahedron by tetrahedron, oriented toward positive phi
__global__ void __launch_bounds__(VOX) mesh_face_kernel(Field F, const unsigned char *__restrict__ mask, const long long *__restrict__ vbase,
							const long long *__restrict__ foff, int *__restrict__ out, long long cap)
{
	__shared__ long long nidx[8], nslot[8];
	__shared__ int warp_s[VOX / 32];
	const long long i = blockIdx.x;
	const int l = threadIdx.x;
	long long b[3];
	brick_of_key(F.key[i], b);
	load_neighbours(F, i, b, nidx, nslot);
	double phi[8];
	const int obs = cube(F, nslot, l, phi);
	int tf;
	long long at = foff[i] + block_scan(face_count(obs, phi), warp_s, &tf);
	for (int t = 0; t < 6; t++) {
		const int nt = tri_count(obs, phi, t);
		if (!nt) continue;
		int cc[4], neg = 0, nm = 0;
		for (int k = 0; k < 4; k++) {
			cc[k] = TET[t][k];
			if (phi[cc[k]] < 0.0) {
				neg |= 1 << k;
				nm++;
			}
		}
		int tri[2][3][2];   // corner pairs (tetrahedron corner indices)
		if (nm == 2) {
			const int a = __ffs(neg) - 1, bb = __ffs(neg & (neg - 1)) - 1;
			const int *o = ORD2[a][bb];
			const int q[2][3][2] = {{{o[0], o[2]}, {o[0], o[3]}, {o[1], o[3]}}, {{o[0], o[2]}, {o[1], o[3]}, {o[1], o[2]}}};
			for (int x = 0; x < 2; x++)
				for (int y = 0; y < 3; y++)
					for (int z = 0; z < 2; z++) tri[x][y][z] = q[x][y][z];
		} else {
			const int lone = nm == 1 ? __ffs(neg) - 1 : __ffs(~neg & 15) - 1;
			const int *o = ORD1[lone];
			const int r1 = nm == 1 ? 2 : 3, r2 = nm == 1 ? 3 : 2;   // a lone positive corner: the other way round
			tri[0][0][0] = tri[0][1][0] = tri[0][2][0] = o[0];
			tri[0][0][1] = o[1];
			tri[0][1][1] = o[r1];
			tri[0][2][1] = o[r2];
		}
		for (int x = 0; x < nt; x++) {
			int idx[3];
			for (int y = 0; y < 3; y++) {
				int lo = cc[tri[x][y][0]], hi = cc[tri[x][y][1]];
				if (__popc(lo) > __popc(hi)) {
					const int s = lo;
					lo = hi;
					hi = s;
				}
				int ll;
				const long long owner = nidx[corner(l, lo, &ll)];
				const int d = DIR_OF[hi ^ lo];
				idx[y] = (int)(vbase[owner * VOX + ll] + __popc(mask[owner * VOX + ll] & ((1u << d) - 1u)));
			}
			if (TET_ODD[t]) {
				const int s = idx[1];
				idx[1] = idx[2];
				idx[2] = s;
			}
			if (at < cap)
				for (int y = 0; y < 3; y++) out[3 * at + y] = idx[y];
			at++;
		}
	}
}

// ---- ray casting ----

__device__ __forceinline__ unsigned long long hash_of(u64 k, int bits) { return (k * 0x9E3779B97F4A7C15ull) >> (64 - bits); }

__global__ void hash_build_kernel(const u64 *__restrict__ key, const long long *__restrict__ slot, long long n, u64 *hkey,
				  long long *hslot, int bits)
{
	const unsigned long long mask = (1ull << bits) - 1;
	for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		const u64 k = key[i];
		for (unsigned long long h = hash_of(k, bits);; h = (h + 1) & mask) {
			if (atomicCAS(hkey + h, EMPTY, k) == EMPTY) {
				hslot[h] = slot[i];
				break;
			}
		}
	}
}

__device__ __forceinline__ long long hash_find(const u64 *hkey, const long long *hslot, int bits, u64 k)
{
	const unsigned long long mask = (1ull << bits) - 1;
	for (unsigned long long h = hash_of(k, bits);; h = (h + 1) & mask) {
		const u64 x = hkey[h];
		if (x == k) return hslot[h];
		if (x == EMPTY) return -1;
	}
}

// phi at world point w by trilinear interpolation over the 8 surrounding voxel centres, false unless all are observed
__device__ __forceinline__ bool sample(const Field &F, const u64 *hkey, const long long *hslot, int bits, const double *w, double *out)
{
	double g[3], fr[3];
	long long i0[3];
	for (int a = 0; a < 3; a++) {
		g[a] = floor(__dsub_rn(__ddiv_rn(w[a], F.v), 0.5));
		if (!(g[a] >= -8.0 * KEY_HALF && g[a] < 8.0 * KEY_HALF - 1.0)) return false;
		fr[a] = __dsub_rn(__dsub_rn(__ddiv_rn(w[a], F.v), 0.5), g[a]);
		i0[a] = (long long)g[a];
	}
	double phi[8];
	u64 last = EMPTY;
	long long s = -1;
	for (int o = 0; o < 8; o++) {
		long long vi[3], bi[3];
		for (int a = 0; a < 3; a++) {
			vi[a] = i0[a] + ((o >> a) & 1);
			bi[a] = vi[a] >> 3;
		}
		u64 k;
		if (!key_of_brick(bi, &k)) return false;
		if (k != last) {
			s = hash_find(hkey, hslot, bits, k);
			last = k;
		}
		const int l = (int)(((vi[2] & 7) << 6) | ((vi[1] & 7) << 3) | (vi[0] & 7));
		if (!phi_at(F, s, l, phi + o)) return false;
	}
	// along x, then y, then z: a + f (b - a)
	double c4[4], c2[2];
	for (int k = 0; k < 4; k++) c4[k] = __dadd_rn(phi[2 * k], __dmul_rn(fr[0], __dsub_rn(phi[2 * k + 1], phi[2 * k])));
	for (int k = 0; k < 2; k++) c2[k] = __dadd_rn(c4[2 * k], __dmul_rn(fr[1], __dsub_rn(c4[2 * k + 1], c4[2 * k])));
	*out = __dadd_rn(c2[0], __dmul_rn(fr[2], __dsub_rn(c2[1], c2[0])));
	return true;
}

__global__ void render_kernel(Field F, const u64 *__restrict__ hkey, const long long *__restrict__ hslot, int bits, int H, int W, Cam c,
			      Pose T, long long kmax, float *__restrict__ depth)
{
	const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= (long)H * W) return;
	const int y = (int)(p / W), x = (int)(p - (long)y * W);
	float Z = CUDART_NAN_F;
	bool prev = false;
	double phi_prev = 0.0;
	float z_prev = 0.f;
	for (long long k = 1; k <= kmax; k++) {
		const float z = __double2float_rn(__dmul_rn((double)k, F.v));
		if (!(z <= c.max_depth)) break;
		double w[3], phi;
		to_world(lateral(x, c.cx, z, c.f), lateral(y, c.cy, z, c.f), z, T, w);
		const bool ok = sample(F, hkey, hslot, bits, w, &phi);
		if (ok && prev && phi_prev >= 0.0 && phi < 0.0) {
			Z = __double2float_rn(__dadd_rn((double)z_prev, __ddiv_rn(__dmul_rn(F.v, phi_prev), __dsub_rn(phi_prev, phi))));
			break;
		}
		prev = ok;
		phi_prev = phi;
		z_prev = z;
	}
	depth[p] = Z;
}

__global__ void table_kernel(const u64 *__restrict__ key, const long long *__restrict__ slot, long long n, char *pool, u64 *keys,
			     double *S, int *nn, int *nc, int *col)
{
	const long long i = blockIdx.x;
	const int l = threadIdx.x;
	const long long s = slot[i], e = i * VOX + l;
	if (l == 0) keys[i] = key[i];
	S[e] = b_S(pool, s)[l];
	nn[e] = b_n(pool, s)[l];
	nc[e] = b_nc(pool, s)[l];
	for (int a = 0; a < 3; a++) col[3 * e + a] = b_col(pool, s, a)[l];
}

}  // namespace

struct mccnn_tsdf {
	double voxel, trunc;
	int K, device;
	long long frames;
	long long n;                  // bricks in the table and the pool
	int cur;                      // key[cur] / slot[cur] hold the table, the other half receives the next merge
	u64 *key[2];
	long long *slot[2], kcap[2];
	char *pool;
	long long pcap;               // bricks the pool holds
	long long *dbox;              // brick-index bounds on the device (min xyz, max xyz), valid when n > 0
	// per-frame scratch, sized for `m` allocation points
	long m;
	void *scratch;
	u64 *keyA, *keyB, *uniq;
	int *valA, *valB, *blk, *hist;
	long long *off, *hoff, *lb, *nn;
	unsigned long long *ctr;
};

namespace {

int grow_scratch(mccnn_tsdf *h, long m)
{
	if (m <= h->m) return 0;
	const long nblk = adc_div_up(m, CHUNK);
	const size_t bytes = 3 * 8 * (size_t)m + 2 * 4 * (size_t)m + 4 * (size_t)nblk + 4 * (size_t)BINS * nblk + 8 * (size_t)(nblk + 1) +
			     8 * (size_t)(BINS * nblk + 1) + 2 * 8 * (size_t)m + 8 * C_N + 128;
	if (h->scratch) ADC_CUDA(cudaFree(h->scratch));
	h->scratch = nullptr;
	h->m = 0;
	ADC_CUDA(cudaMalloc(&h->scratch, bytes));
	char *p = (char *)h->scratch;
	auto take = [&p](size_t b) {
		char *q = p;
		p += (b + 7) & ~(size_t)7;
		return q;
	};
	h->keyA = (u64 *)take(8 * (size_t)m);
	h->keyB = (u64 *)take(8 * (size_t)m);
	h->uniq = (u64 *)take(8 * (size_t)m);
	h->lb = (long long *)take(8 * (size_t)m);
	h->nn = (long long *)take(8 * (size_t)m);
	h->off = (long long *)take(8 * (size_t)(nblk + 1));
	h->hoff = (long long *)take(8 * (size_t)(BINS * nblk + 1));
	h->ctr = (unsigned long long *)take(8 * C_N);
	h->valA = (int *)take(4 * (size_t)m);
	h->valB = (int *)take(4 * (size_t)m);
	h->blk = (int *)take(4 * (size_t)nblk);
	h->hist = (int *)take(4 * (size_t)BINS * nblk);
	h->m = m;
	return 0;
}

// makes key / slot half `k` hold at least `need` bricks; its contents are not kept
int reserve_keys(mccnn_tsdf *h, int k, long long need)
{
	if (h->key[k] && h->kcap[k] >= need) return 0;
	const long long cap = std::max<long long>(need + need / 2, 1024);
	if (h->key[k]) ADC_CUDA(cudaFree(h->key[k]));
	h->key[k] = nullptr;
	ADC_CUDA(cudaMalloc(&h->key[k], 16 * (size_t)cap));
	h->slot[k] = (long long *)(h->key[k] + cap);
	h->kcap[k] = cap;
	return 0;
}

// makes the pool hold at least `need` bricks, keeping the first h->n
int reserve_pool(mccnn_tsdf *h, long long need, cudaStream_t s)
{
	if (h->pool && h->pcap >= need) return 0;
	const long long cap = std::max<long long>(need + need / 2, 256);
	char *p = nullptr;
	ADC_CUDA(cudaMalloc(&p, (size_t)cap * BRICK_BYTES));
	if (h->pool) {
		cudaError_t e = cudaMemcpyAsync(p, h->pool, (size_t)h->n * BRICK_BYTES, cudaMemcpyDeviceToDevice, s);
		if (e == cudaSuccess) e = cudaStreamSynchronize(s);
		if (e != cudaSuccess) {
			cudaFree(p);
			return (int)e;
		}
		ADC_CUDA(cudaFree(h->pool));
	}
	h->pool = p;
	h->pcap = cap;
	return 0;
}

Field field_of(const mccnn_tsdf *h, int min_frames)
{
	return Field{h->key[h->cur], h->slot[h->cur], h->n, h->pool, h->voxel, min_frames};
}

int run_add(mccnn_tsdf *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, const Cam &c, const Pose &T,
	    long long *stats, cudaStream_t s)
{
	const int J = 2 * h->K + 1;
	const long m = (long)H * W * J;
	const int nblk = adc_div_up(m, CHUNK);
	int rc = grow_scratch(h, m);
	if (rc) return rc;
	const float step = (float)(h->trunc / h->K);
	ADC_CUDA(cudaMemsetAsync(h->ctr, 0, 8 * C_N, s));
	long long *ctr = (long long *)h->ctr;
	// 1. allocation: the ray points' brick keys, sorted, one per run, ranked in the table
	alloc_count_kernel<<<nblk, THREADS, 0, s>>>(disp, m, J, W, c, T, step, h->voxel, h->blk, h->ctr);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_M);
	alloc_fill_kernel<<<nblk, THREADS, 0, s>>>(disp, m, J, W, c, T, step, h->voxel, h->off, h->keyA, h->valA);
	ADC_CHECK_LAUNCH();
	radix_sort_pairs(h->keyA, h->valA, h->keyB, h->valB, ctr + C_M, nblk, h->hist, h->hoff, ctr + C_SCRATCH, s);
	head_count_kernel<<<nblk, THREADS, 0, s>>>(h->keyA, ctr + C_M, h->blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_U);
	head_fill_kernel<<<nblk, THREADS, 0, s>>>(h->keyA, ctr + C_M, h->off, h->uniq);
	const long long tn = h->n;
	const u64 *tkey = tn ? h->key[h->cur] : nullptr;
	match_count_kernel<<<nblk, THREADS, 0, s>>>(h->uniq, ctr + C_U, tkey, tn, h->lb, h->blk);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(h->blk, nblk, h->off, ctr + C_NEW);
	match_rank_kernel<<<nblk, THREADS, 0, s>>>(h->uniq, ctr + C_U, tkey, tn, h->lb, h->off, h->nn);
	ADC_CHECK_LAUNCH();
	long long nnew = 0;
	ADC_CUDA(cudaMemcpyAsync(&nnew, ctr + C_NEW, sizeof nnew, cudaMemcpyDeviceToHost, s));
	ADC_CUDA(cudaStreamSynchronize(s));
	const int dst = 1 - h->cur;
	if ((rc = reserve_keys(h, dst, tn + nnew)) || (rc = reserve_pool(h, tn + nnew, s))) return rc;
	if (nnew) {
		ADC_CUDA(cudaMemsetAsync(h->pool + tn * BRICK_BYTES, 0, (size_t)nnew * BRICK_BYTES, s));
		if (tn)
			merge_table_kernel<<<grid_for(tn), THREADS, 0, s>>>(h->key[h->cur], h->slot[h->cur], tn, h->uniq, ctr + C_U, h->nn,
									     ctr + C_NEW, h->key[dst], h->slot[dst]);
		merge_frame_kernel<<<grid_for(m), THREADS, 0, s>>>(h->uniq, ctr + C_U, h->lb, h->nn, tkey, tn, h->key[dst], h->slot[dst],
								     h->dbox);
		ADC_CHECK_LAUNCH();
		h->cur = dst;
		h->n = tn + nnew;
	}
	ADC_CUDA(cudaMemcpyAsync(stats, ctr + C_PIX, 8, cudaMemcpyDeviceToDevice, s));
	ADC_CUDA(cudaMemcpyAsync(stats + 1, ctr + C_OUT, 8, cudaMemcpyDeviceToDevice, s));
	// 2. integration over every brick of the table
	if (h->n)
		integrate_kernel<<<(unsigned)h->n, VOX, 0, s>>>(h->key[h->cur], h->slot[h->cur], h->pool, disp, rgb, nch, c,
								 Proj{H, W, (double)c.f, (double)c.cx, (double)c.cy}, T, h->voxel, h->trunc);
	ADC_CHECK_LAUNCH();
	h->frames++;
	return 0;
}

bool camera_ok(float f, float cx, float cy, float max_depth)
{
	return f > 0.f && isfinite(f) && isfinite(cx) && isfinite(cy) && max_depth > 0.f;
}

// the largest camera depth of a point in the brick-index bounds `box` (a linear function of the point: a corner's), for
// the pose's inverse, plus a margin; +inf when R is singular.  A valid sample lies inside the bounds, so a ray ends there.
double far_depth(const mccnn_tsdf *h, const long long *box, const Pose &T)
{
	const double *r = T.r;
	const double a = r[0], b = r[1], c = r[2], d = r[4], e = r[5], f = r[6], g = r[8], k = r[9], l = r[10];
	const double det = a * (e * l - f * k) - b * (d * l - f * g) + c * (d * k - e * g);
	if (!(det != 0.0) || !isfinite(det)) return INFINITY;
	const double row[3] = {(d * k - e * g) / det, -(a * k - b * g) / det, (a * e - b * d) / det};   // the inverse's last row
	const double lo = 8.0 * h->voxel, v = h->voxel;
	double zmax = -INFINITY;
	for (int o = 0; o < 8; o++) {
		double z = 0.0;
		for (int x = 0; x < 3; x++) {
			const double w = (o >> x & 1) ? (box[3 + x] + 1) * lo : box[x] * lo;
			z += row[x] * (w - r[4 * x + 3]);
		}
		zmax = std::max(zmax, z);
	}
	if (!isfinite(zmax)) return INFINITY;
	return zmax + 1e-6 * fabs(zmax) + 2.0 * v;
}

}  // namespace

extern "C" {

int mccnn_tsdf_create(mccnn_tsdf **out, double voxel, double trunc, int device)
{
	if (!out) return ADCENSUS_EINVAL;
	*out = nullptr;
	if (!(voxel > 0.0) || !isfinite(voxel) || !isfinite(trunc) || !(trunc >= voxel)) return ADCENSUS_EINVAL;
	const double K = ceil(trunc / (4.0 * voxel));
	if (K > 64) return ADCENSUS_ELIMIT;
	int ndev = 0;
	ADC_CUDA(cudaGetDeviceCount(&ndev));
	if (device < 0 || device >= ndev) return ADCENSUS_EINVAL;
	DeviceScope dev(device);
	if (dev.rc) return dev.rc;
	long long *dbox = nullptr;
	ADC_CUDA(cudaMalloc(&dbox, sizeof(long long) * 6));
	const long long init[6] = {KEY_HALF, KEY_HALF, KEY_HALF, -KEY_HALF - 1, -KEY_HALF - 1, -KEY_HALF - 1};
	const cudaError_t e = cudaMemcpy(dbox, init, sizeof init, cudaMemcpyHostToDevice);
	if (e != cudaSuccess) {
		cudaFree(dbox);
		return (int)e;
	}
	mccnn_tsdf *h = new mccnn_tsdf();
	h->voxel = voxel;
	h->trunc = trunc;
	h->K = (int)K;
	h->device = device;
	h->dbox = dbox;
	*out = h;
	return 0;
}

int mccnn_tsdf_add(mccnn_tsdf *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy,
		   float fB, float doffs, float max_depth, const double *pose12, long long *stats, adcensus_stream_t stream)
{
	if (!h || !disp || !rgb || !stats || (nch != 1 && nch != 3) || H < 1 || W < 1) return ADCENSUS_EINVAL;
	if ((long)H * W * nch >= (1l << 31) || (long)H * W * (2 * h->K + 1) >= (1l << 31) || h->frames >= MAX_FRAMES)
		return ADCENSUS_ELIMIT;
	if (!(camera_ok(f, cx, cy, max_depth) && fB > 0.f && isfinite(fB) && isfinite(doffs))) return ADCENSUS_EINVAL;
	Pose T;
	int rc = check_pose(pose12, &T);
	if (rc) return rc;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	return run_add(h, disp, rgb, nch, H, W, Cam{f, cx, cy, fB, doffs, max_depth}, T, stats, adc_stream(stream));
}

long long mccnn_tsdf_bricks(const mccnn_tsdf *h) { return h ? h->n : -1; }

long long mccnn_tsdf_pool_bytes(const mccnn_tsdf *h) { return h ? h->pcap * BRICK_BYTES : -1; }

int mccnn_tsdf_table(const mccnn_tsdf *h, unsigned long long *keys, double *S, int *n, int *nc, int *colours, adcensus_stream_t stream)
{
	if (!h) return ADCENSUS_EINVAL;
	if (!h->n) return 0;
	if (!keys || !S || !n || !nc || !colours) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	table_kernel<<<(unsigned)h->n, VOX, 0, adc_stream(stream)>>>(h->key[h->cur], h->slot[h->cur], h->n, h->pool, keys, S, n, nc,
								     colours);
	return (int)cudaPeekAtLastError();
}

int mccnn_tsdf_mesh_count(const mccnn_tsdf *h, int min_frames, long long *counts, adcensus_stream_t stream)
{
	if (!h || !counts || min_frames < 1) return ADCENSUS_EINVAL;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	const long long n = h->n;
	if (!n) return (int)cudaMemsetAsync(counts, 0, 2 * sizeof(long long), s);
	void *mem = nullptr;
	int rc = adc_scratch_alloc(&mem, (size_t)n * VOX + 8 * (size_t)(4 * n + 2), s);
	if (rc) return rc;
	long long *off = (long long *)mem;
	int *vb = (int *)(off + 2 * n), *fb = vb + n;
	unsigned char *mask = (unsigned char *)(fb + n);
	const Field F = field_of(h, min_frames);
	mesh_count_kernel<<<(unsigned)n, VOX, 0, s>>>(F, mask, vb, fb);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(vb, n, off, counts);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(fb, n, off + n, counts + 1);
	rc = (int)cudaPeekAtLastError();
	const int rf = adc_scratch_free(mem, s);
	return rc ? rc : rf;
}

int mccnn_tsdf_mesh_fill(const mccnn_tsdf *h, int min_frames, unsigned char *verts, long long vcap, int *faces, long long fcap,
			 adcensus_stream_t stream)
{
	if (!h || min_frames < 1 || vcap < 0 || fcap < 0 || (vcap && !verts) || (fcap && !faces)) return ADCENSUS_EINVAL;
	if (vcap >= (1ll << 31)) return ADCENSUS_ELIMIT;
	const long long n = h->n;
	if (!n || (!vcap && !fcap)) return 0;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	void *mem = nullptr;
	int rc = adc_scratch_alloc(&mem, 8 * (size_t)n * VOX + (size_t)n * VOX + 8 * (size_t)(4 * n + 2), s);
	if (rc) return rc;
	long long *vbase = (long long *)mem, *off = vbase + n * VOX;
	int *vb = (int *)(off + 2 * n + 2), *fb = vb + n;
	unsigned char *mask = (unsigned char *)(fb + n);
	const Field F = field_of(h, min_frames);
	mesh_count_kernel<<<(unsigned)n, VOX, 0, s>>>(F, mask, vb, fb);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(vb, n, off, off + 2 * n);
	scan_kernel<<<1, SCAN_THREADS, 0, s>>>(fb, n, off + n, off + 2 * n + 1);
	mesh_vertex_kernel<<<(unsigned)n, VOX, 0, s>>>(F, mask, off, vbase, verts, vcap);
	mesh_face_kernel<<<(unsigned)n, VOX, 0, s>>>(F, mask, vbase, off + n, faces, fcap);
	rc = (int)cudaPeekAtLastError();
	const int rf = adc_scratch_free(mem, s);
	return rc ? rc : rf;
}

int mccnn_tsdf_render(const mccnn_tsdf *h, int min_frames, int H, int W, float f, float cx, float cy, float max_depth,
		      const double *pose12, float *depth, adcensus_stream_t stream)
{
	if (!h || !depth || min_frames < 1 || H < 1 || W < 1 || !camera_ok(f, cx, cy, max_depth)) return ADCENSUS_EINVAL;
	if ((long)H * W >= (1l << 31)) return ADCENSUS_ELIMIT;
	Pose T;
	int rc = check_pose(pose12, &T);
	if (rc) return rc;
	DeviceScope dev(h->device);
	if (dev.rc) return dev.rc;
	cudaStream_t s = adc_stream(stream);
	long long box[6];
	ADC_CUDA(cudaMemcpyAsync(box, h->dbox, sizeof box, cudaMemcpyDeviceToHost, s));
	ADC_CUDA(cudaStreamSynchronize(s));
	const double zfar = h->n ? std::min<double>(max_depth, far_depth(h, box, T)) : 0.0;
	if (!isfinite(zfar)) return ADCENSUS_EINVAL;
	const long long kmax = (long long)ceil(zfar / h->voxel) + 1;
	int bits = 10;
	while ((1ll << bits) < 2 * h->n) bits++;
	void *mem = nullptr;
	rc = adc_scratch_alloc(&mem, 16ull << bits, s);
	if (rc) return rc;
	u64 *hkey = (u64 *)mem;
	long long *hslot = (long long *)(hkey + (1ll << bits));
	rc = (int)cudaMemsetAsync(hkey, 0xff, 8ull << bits, s);
	if (!rc && h->n) hash_build_kernel<<<grid_for(h->n), THREADS, 0, s>>>(h->key[h->cur], h->slot[h->cur], h->n, hkey, hslot, bits);
	const long npx = (long)H * W;
	if (!rc)
		render_kernel<<<adc_div_up(npx, THREADS), THREADS, 0, s>>>(field_of(h, min_frames), hkey, hslot, bits, H, W,
									   Cam{f, cx, cy, 1.f, 0.f, max_depth}, T, h->n ? kmax : 0, depth);
	if (!rc) rc = (int)cudaPeekAtLastError();
	const int rf = adc_scratch_free(mem, s);
	return rc ? rc : rf;
}

void mccnn_tsdf_destroy(mccnn_tsdf *h)
{
	if (!h) return;
	{
		DeviceScope dev(h->device);
		if (!dev.rc) {
			for (void *p : {(void *)h->key[0], (void *)h->key[1], (void *)h->pool, h->scratch, (void *)h->dbox})
				if (p) cudaFree(p);
		}
	}
	delete h;
}

}  // extern "C"
