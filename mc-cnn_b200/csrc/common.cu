// common.cu -- device properties cache, stream-ordered scratch, shared-memory opt-in, version string
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"

namespace {

// ADCENSUS_NUM_SMS as a decimal integer in 1..1024, or 0 when it is unset or anything else (DESIGN §4)
int forced_num_sms()
{
	const char *v = getenv("ADCENSUS_NUM_SMS");
	if (!v || !*v || strlen(v) > 4) return 0;
	int n = 0;
	for (const char *c = v; *c; c++) {
		if (*c < '0' || *c > '9') return 0;
		n = 10 * n + (*c - '0');
	}
	return n >= 1 && n <= 1024 ? n : 0;
}

}  // namespace

int adc_num_sms()
{
	static int sms[64] = {0};
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) return 132;
	if (!sms[dev & 63]) {
		static const int forced = forced_num_sms();
		int n = forced;
		if (!n && (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)) n = 132;
		sms[dev & 63] = n;
	}
	return sms[dev & 63];
}

int adc_scratch_alloc(void **p, size_t bytes, cudaStream_t s)
{
	// keep freed scratch in the device's default pool instead of returning it to the OS at every
	// synchronisation (the default release threshold is 0), so repeated op-level calls reuse it
	static bool tuned[64] = {false};
	int dev = 0;
	if (cudaGetDevice(&dev) == cudaSuccess && !tuned[dev & 63]) {
		cudaMemPool_t pool;
		if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
			// bounded: a drop-in library must not pin unlimited memory in a pool the host application (torch's
			// caching allocator, cutorch) cannot reuse; adcensus_trim_scratch() returns it on demand
			unsigned long long keep = 2ULL << 30, cur = 0;
			cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &cur);
			if (cur < keep) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
		}
		tuned[dev & 63] = true;
	}
	return (int)cudaMallocAsync(p, bytes ? bytes : 4, s);
}

int adc_scratch_free(void *p, cudaStream_t s)
{
	return p ? (int)cudaFreeAsync(p, s) : 0;
}

// The attribute only ever grows: a launch that needs less than an earlier one must not lower it under a launch of
// another host thread.  `granted` is the record per (device, kernel), written under the lock; each host thread keeps a
// copy of what it has read there, so a launch whose amount is already granted takes no lock.
int adc_smem_optin(const void *kernel, size_t bytes)
{
	if (bytes <= 48 * 1024) return 0;
	if (bytes > 232448) return ADCENSUS_ELIMIT;
	int dev = 0;
	ADC_CUDA(cudaGetDevice(&dev));
	const std::pair<int, const void *> key(dev, kernel);
	thread_local std::map<std::pair<int, const void *>, size_t> seen;
	const auto it = seen.find(key);
	if (it != seen.end() && it->second >= bytes) return 0;
	static std::mutex mu;
	static std::map<std::pair<int, const void *>, size_t> granted;
	std::lock_guard<std::mutex> lock(mu);
	size_t &g = granted[key];
	if (g < bytes) {
		ADC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
		g = bytes;
	}
	seen[key] = g;
	return 0;
}

// give the stream-ordered scratch kept by the operator-level calls back to the driver (after the work using it has completed)
extern "C" int adcensus_trim_scratch(void)
{
	int dev = 0;
	cudaMemPool_t pool;
	ADC_CUDA(cudaGetDevice(&dev));
	ADC_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
	ADC_CUDA(cudaMemPoolTrimTo(pool, 0));
	return 0;
}

extern "C" const char *adcensus_version(void) { return "libadcensus_b200 0.1.0 (sm_90a)"; }

extern "C" int adcensus_num_sms(void) { return adc_num_sms(); }

// ---------------------------------------------------------------- TMA tensor maps
#include "tma.cuh"

typedef CUresult (*adc_encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
					const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
					CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static adc_encode_tiled_fn adc_encode_tiled()
{
	static adc_encode_tiled_fn fn = nullptr;
	static bool tried = false;
	if (!tried) {
		void *p = nullptr;
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
		    q == cudaDriverEntryPointSuccess)
			fn = (adc_encode_tiled_fn)p;
		tried = true;
	}
	return fn;
}

int adc_tma_encode(CUtensorMap *map, const void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
		   const uint32_t *box)
{
	adc_encode_tiled_fn fn = adc_encode_tiled();
	if (!fn) return (int)cudaErrorNotSupported;
	if (rank < 2 || rank > 3 || ((uintptr_t)base & 15)) return ADCENSUS_EINVAL;
	cuuint64_t gd[3], gs[2];
	cuuint32_t bx[3], es[3] = {1, 1, 1};
	for (int i = 0; i < rank; i++) { gd[i] = dims[i]; bx[i] = box[i]; }
	for (int i = 0; i + 1 < rank; i++) {
		if (strides_bytes[i] % 16) return ADCENSUS_EINVAL;
		gs[i] = strides_bytes[i];
	}
	CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), gd, gs, bx, es,
			CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
			CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}
