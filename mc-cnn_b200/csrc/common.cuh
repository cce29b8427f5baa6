// common.cuh -- shared helpers for the sm_90a kernels of libadcensus_b200.so
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "adcensus_b200.h"

#define ADC_CHECK_LAUNCH()                                   \
	do {                                                 \
		cudaError_t e__ = cudaPeekAtLastError();     \
		if (e__ != cudaSuccess) return (int)e__;     \
	} while (0)

#define ADC_CUDA(call)                                       \
	do {                                                 \
		cudaError_t e__ = (call);                    \
		if (e__ != cudaSuccess) return (int)e__;     \
	} while (0)

static inline cudaStream_t adc_stream(adcensus_stream_t s) { return (cudaStream_t)s; }

static inline int adc_div_up(long a, long b) { return (int)((a + b - 1) / b); }

// makes `device` current for the scope of one call and restores the caller's device
struct DeviceScope {
	int prev = -1;
	int rc = 0;
	explicit DeviceScope(int device)
	{
		rc = (int)cudaGetDevice(&prev);
		if (!rc && prev != device) rc = (int)cudaSetDevice(device);
	}
	~DeviceScope()
	{
		if (prev >= 0) cudaSetDevice(prev);
	}
};

// number of SMs of the current device (cached per device; 132 on H100 SXM)
int adc_num_sms();

// stream-ordered scratch (cudaMallocAsync on the device's default pool)
int adc_scratch_alloc(void **p, size_t bytes, cudaStream_t s);
int adc_scratch_free(void *p, cudaStream_t s);

// Lets `kernel` launch on the current device with `bytes` of dynamic shared memory: nothing to do up to 48 KB,
// ADCENSUS_ELIMIT above the 227 KB per-block limit of sm_90.  Safe to call from several host threads and cheap on
// every launch once the amount has been granted.
int adc_smem_optin(const void *kernel, size_t bytes);
template <typename Kernel>
int adc_smem_optin(Kernel *kernel, size_t bytes)
{
	return adc_smem_optin((const void *)kernel, bytes);
}

__device__ __forceinline__ float adc_nan() { return __int_as_float(0x7fffffff); }

// streaming (evict-first) global accesses for data touched exactly once
__device__ __forceinline__ float ld_stream(const float *p)
{
	float v;
	asm volatile("ld.global.cs.f32 %0, [%1];" : "=f"(v) : "l"(p));
	return v;
}
__device__ __forceinline__ void st_stream(float *p, float v)
{
	asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v));
}
