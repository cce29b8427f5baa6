// pairwise.cuh -- numpy's pairwise summation (pairwise_sum of numpy's umath loops) reproduced on the GPU, for every kernel
// that must give the bits of a numpy sum over a contiguous array: float32 (x.mean() / x.std() of a float32 array) or
// float64 (x.astype(np.float64).sum()) accumulation, and any per-element transform.
//
// numpy's order over n elements in memory order: n > 128 splits into [0, n2) and [n2, n), n2 = n / 2 rounded down to a
// multiple of 8, and the two halves' sums are added; a leaf of n < 8 elements is summed in turn from 0; a leaf of 8..128
// elements runs eight strided accumulators r[j] (element j, then += element i + j for i = 8, 16, ...), combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), and the remainder added in turn.  Every add is one IEEE add in the
// accumulation type.  One thread per leaf, then the internal nodes level by level in one block per view: deterministic.
#pragma once

#include <vector>

#include "common.cuh"

namespace pairwise {

constexpr int LEAF = 128;                 // numpy's PW_BLOCKSIZE
constexpr int COMBINE_THREADS = 1024;
constexpr int LEAF_THREADS = 256;

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// leaf k of view blockIdx.y: the sum of elem(view, i) over the leaf's elements, into val[view * nval + k]
template <typename T, class Elem>
__global__ void leaf_kernel(Elem elem, const int2 *__restrict__ leaves, int nleaf, int nval, T *__restrict__ val)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= nleaf) return;
	const int view = blockIdx.y;
	const long a = leaves[k].x;
	const int n = leaves[k].y;
	T res = 0;
	if (n < 8) {
		for (int i = 0; i < n; i++) res = add_rn(res, elem(view, a + i));
	} else {
		T r[8];
#pragma unroll
		for (int j = 0; j < 8; j++) r[j] = elem(view, a + j);
		const int body = n - n % 8;
		for (int i = 8; i < body; i += 8) {
#pragma unroll
			for (int j = 0; j < 8; j++) r[j] = add_rn(r[j], elem(view, a + i + j));
		}
		res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
		for (int i = body; i < n; i++) res = add_rn(res, elem(view, a + i));
	}
	val[(long)view * nval + k] = res;
}

// The internal nodes sorted by height: level h (1..) holds the nodes lev_off[h-1] .. lev_off[h]-1 (ids nleaf + index), each
// the sum of its two children.  The root is the last node; fin(view, root) runs once per view.
template <typename T, class Finish>
__global__ void __launch_bounds__(COMBINE_THREADS) combine_kernel(const int2 *__restrict__ child, const int *__restrict__ lev_off,
								  int nlev, int nleaf, int nval, T *__restrict__ val, Finish fin)
{
	T *v = val + (long)blockIdx.x * nval;
	for (int h = 0; h < nlev; h++) {
		for (int k = lev_off[h] + threadIdx.x; k < lev_off[h + 1]; k += COMBINE_THREADS)
			v[nleaf + k] = add_rn(v[child[k].x], v[child[k].y]);
		__syncthreads();
	}
	if (threadIdx.x == 0) fin(blockIdx.x, v[nval - 1]);
}

// The tree of `count` elements for `nviews` views in stream-ordered scratch.  init() builds and uploads it, each sum() is
// one leaf and one combine launch (all views at once), release() frees the scratch in stream order.  count < 2^31.
template <typename T>
class Sum {
public:
	int init(long count, int nviews, cudaStream_t s)
	{
		s_ = s;
		nviews_ = nviews;
		std::vector<int2> leaves;
		std::vector<std::vector<int4>> levels;      // per height - 1: (left height, left index, right height, right index)
		build(0, count, leaves, levels);
		nleaf_ = (int)leaves.size();
		std::vector<int> lev_off(1, 0);
		for (auto &l : levels) lev_off.push_back(lev_off.back() + (int)l.size());
		const int ninner = lev_off.back();
		nlev_ = (int)levels.size();
		std::vector<int2> child(ninner);
		auto id = [&](int h, int k) { return h == 0 ? k : nleaf_ + lev_off[h - 1] + k; };
		for (int h = 1; h <= nlev_; h++)
			for (size_t k = 0; k < levels[h - 1].size(); k++) {
				const int4 c = levels[h - 1][k];
				child[lev_off[h - 1] + k] = make_int2(id(c.x, c.y), id(c.z, c.w));
			}
		nval_ = nleaf_ + ninner;

		// the value array first, padded to 16 bytes so that the int2 arrays after it are aligned
		const size_t b_val = (sizeof(T) * (size_t)nval_ * nviews + 15) & ~(size_t)15, b_leaves = sizeof(int2) * nleaf_,
			     b_child = sizeof(int2) * (ninner + 1), b_lev = sizeof(int) * lev_off.size();
		int rc = adc_scratch_alloc((void **)&scratch_, b_val + b_leaves + b_child + b_lev, s);
		if (rc) return rc;
		val_ = (T *)scratch_;
		leaves_ = (int2 *)(scratch_ + b_val);
		child_ = (int2 *)(scratch_ + b_val + b_leaves);
		lev_ = (int *)(scratch_ + b_val + b_leaves + b_child);
		// pageable sources: cudaMemcpyAsync returns once they are staged, so the vectors may go out of scope
		cudaError_t e = cudaMemcpyAsync(leaves_, leaves.data(), b_leaves, cudaMemcpyHostToDevice, s);
		if (e == cudaSuccess && ninner)
			e = cudaMemcpyAsync(child_, child.data(), sizeof(int2) * ninner, cudaMemcpyHostToDevice, s);
		if (e == cudaSuccess) e = cudaMemcpyAsync(lev_, lev_off.data(), b_lev, cudaMemcpyHostToDevice, s);
		return (int)e;
	}

	template <class Elem, class Finish>
	int sum(const Elem &elem, const Finish &fin)
	{
		const dim3 grid((nleaf_ + LEAF_THREADS - 1) / LEAF_THREADS, nviews_);
		leaf_kernel<T><<<grid, LEAF_THREADS, 0, s_>>>(elem, leaves_, nleaf_, nval_, val_);
		combine_kernel<T><<<nviews_, COMBINE_THREADS, 0, s_>>>(child_, lev_, nlev_, nleaf_, nval_, val_, fin);
		return (int)cudaPeekAtLastError();
	}

	int release() { return scratch_ ? adc_scratch_free(scratch_, s_) : 0; }

private:
	// returns (height, index within that height); height 0 = leaf
	static int2 build(long a, long n, std::vector<int2> &leaves, std::vector<std::vector<int4>> &levels)
	{
		if (n <= LEAF) {
			leaves.push_back(make_int2((int)a, (int)n));
			return make_int2(0, (int)leaves.size() - 1);
		}
		long n2 = n / 2;
		n2 -= n2 % 8;
		const int2 l = build(a, n2, leaves, levels), r = build(a + n2, n - n2, leaves, levels);
		const int h = (l.x > r.x ? l.x : r.x) + 1;
		if ((int)levels.size() < h) levels.resize(h);
		levels[h - 1].push_back(make_int4(l.x, l.y, r.x, r.y));
		return make_int2(h, (int)levels[h - 1].size() - 1);
	}

	cudaStream_t s_ = nullptr;
	char *scratch_ = nullptr;
	T *val_ = nullptr;
	int2 *leaves_ = nullptr, *child_ = nullptr;
	int *lev_ = nullptr;
	int nviews_ = 0, nleaf_ = 0, nval_ = 0, nlev_ = 0;
};

}  // namespace pairwise
