// render.cu -- the images a user looks at a result with, for sm_90a: samples/bin2png.lua's grey maps of a cost volume and of
// a disparity map, and main.lua -debug's colour images (adcensus.grey2jet and the good / bad pixel tint, main.lua:1240-1265).
//
// Each kernel restates the reference's sequence of tensor operations in the precision its tensors had (float32 for the
// FloatTensor / CudaTensor ops, double where main.lua converts with :double()), then quantises as image.save does.
#include <stdio.h>
#include <sys/types.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr size_t CHUNK_BYTES = 64ul << 20;   // one streaming buffer of mccnn_render_volume_file

// image.save of a float image: image.saturate's clamp to [0, 1], times 255 in double, the byte conversion truncates.
// NaN survives saturate and converts to 0 on x86.
__device__ __forceinline__ unsigned char quantise(double v)
{
	if (!(v > 0.0)) return 0;
	return (unsigned char)__double2int_rz(__dmul_rn(v > 1.0 ? 1.0 : v, 255.0));
}

// fromfile's x[x:ne(x)] = 1e38 (bin2png.lua:13-14), a float32 store
__device__ __forceinline__ float nan_to_big(float v) { return v != v ? 1e38f : v; }

long grid_for(long n) { return std::min<long>((n + THREADS - 1) / THREADS, (long)adc_num_sms() * 8); }

// one chunk of n rows: vol (D, n, W) -> grey of those rows.  left:min(2) with the first index kept on ties, then
// :float():div(D) in fp32 on the 1-based index
__global__ void volume_grey_kernel(const float *__restrict__ vol, int D, long hw, unsigned char *__restrict__ grey)
{
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x) {
		float m = nan_to_big(vol[p]);
		int idx = 0;
		for (int d = 1; d < D; d++) {
			const float v = nan_to_big(vol[(long)d * hw + p]);
			if (v < m) {
				m = v;
				idx = d;
			}
		}
		grey[p] = quantise((double)__fdiv_rn((float)(idx + 1), (float)D));
	}
}

__global__ void map_grey_kernel(const float *__restrict__ x, long hw, float d, unsigned char *__restrict__ grey)
{
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x)
		grey[p] = quantise((double)__fdiv_rn(nan_to_big(x[p]), d));
}

// x:double():add(1):div(disp_max), then grey2jet's val = grey * 4 and its five bands (adcensus.cu:2017-2046)
__global__ void jet_kernel(const float *__restrict__ x, long hw, double disp_max, int mask_blue, unsigned char *__restrict__ rgb,
			   int *__restrict__ refused)
{
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x) {
		const float xv = x[p];
		const double val = __dmul_rn(__ddiv_rn(__dadd_rn((double)xv, 1.0), disp_max), 4.0);
		double r = 0, g = 0, b = 0;
		if (-0.1 <= val && val < 0.5) {
			b = __dadd_rn(0.5, val);
		} else if (0.5 <= val && val < 1.5) {
			g = __dsub_rn(val, 0.5);
			b = 1;
		} else if (1.5 <= val && val < 2.5) {
			r = __dsub_rn(val, 1.5);
			g = 1;
			b = __dsub_rn(1.0, __dsub_rn(val, 1.5));
		} else if (2.5 <= val && val < 3.5) {
			r = 1;
			g = __dsub_rn(1.0, __dsub_rn(val, 2.5));
		} else if (3.5 <= val && val <= 4.1) {
			r = __dsub_rn(1.0, __dsub_rn(val, 3.5));
		} else {
			*refused = 1;     // the reference's assert(0); the pixel stays black
		}
		if (mask_blue) b = __dmul_rn(b, xv != 0.f ? 1.0 : 0.0);   // img_gt[{1,3}]:cmul(mask:double())
		rgb[3 * p] = quantise(r);
		rgb[3 * p + 1] = quantise(g);
		rgb[3 * p + 2] = quantise(b);
	}
}

// main.lua:1243-1252 in fp32; cutorch's div(v) is mul(1 / v) with the reciprocal rounded to float
__global__ void error_kernel(const float *__restrict__ x0, const float *__restrict__ pred, const float *__restrict__ gt, long hw,
			     float err_at, unsigned char *__restrict__ rgb)
{
	const float inv255 = 1.f / 255.f;
	for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long)gridDim.x * blockDim.x) {
		const float grey = __fmul_rn(__fadd_rn(__fmul_rn(x0[p], 50.f), 150.f), inv255);
		const float g = gt[p];
		const float diff = fabsf(__fsub_rn(g, pred[p]));
		const float mask = g != 0.f ? 1.f : 0.f;
		const float bad = __fmul_rn(diff > err_at ? 1.f : 0.f, mask);
		const float good = __fmul_rn(diff <= err_at ? 1.f : 0.f, mask);
		const float r = __fadd_rn(__fadd_rn(grey, __fmul_rn(0.5f, bad)), __fmul_rn(-0.5f, good));
		const float gr = __fadd_rn(__fadd_rn(grey, __fmul_rn(-0.5f, bad)), __fmul_rn(0.5f, good));
		const float b = __fadd_rn(__fadd_rn(grey, __fmul_rn(-0.5f, bad)), __fmul_rn(-0.5f, good));
		rgb[3 * p] = quantise((double)r);
		rgb[3 * p + 1] = quantise((double)gr);
		rgb[3 * p + 2] = quantise((double)b);
	}
}

// the rows [y0, y0 + n) of every disparity plane of the (D, H, W) file into buf (D, n, W)
int read_rows(FILE *f, int D, int H, int W, int y0, int n, float *buf)
{
	const size_t len = (size_t)n * W;
	for (int d = 0; d < D; d++) {
		if (fseeko(f, (off_t)(((long)d * H + y0) * W) * (off_t)sizeof(float), SEEK_SET) != 0) return ADCENSUS_EIO;
		if (fread(buf + (size_t)d * len, sizeof(float), len, f) != len) return ADCENSUS_EIO;
	}
	return 0;
}

}  // namespace

extern "C" int mccnn_render_volume_file(const char *path, int D, int H, int W, unsigned char *grey, adcensus_stream_t stream)
{
	if (!path || !grey || D < 1 || H < 1 || W < 1 || (long)H * W >= (1l << 31)) return ADCENSUS_EINVAL;
	FILE *f = fopen(path, "rb");
	if (!f) return ADCENSUS_EIO;
	if (fseeko(f, 0, SEEK_END) != 0 || ftello(f) < (off_t)D * H * W * (off_t)sizeof(float)) {
		fclose(f);
		return ADCENSUS_EIO;
	}
	const size_t row = (size_t)D * W * sizeof(float);                // one image row over every disparity
	const int rows = (int)std::min<size_t>((size_t)H, std::max<size_t>(1, CHUNK_BYTES / row));
	float *host[2] = {nullptr, nullptr}, *dev[2] = {nullptr, nullptr};
	cudaStream_t st[2] = {nullptr, nullptr};
	cudaEvent_t ready = nullptr;
	int rc = (int)cudaEventCreateWithFlags(&ready, cudaEventDisableTiming);
	if (!rc) rc = (int)cudaEventRecord(ready, adc_stream(stream));   // grey may still be in use by earlier work
	for (int k = 0; k < 2 && !rc; k++) {
		rc = (int)cudaStreamCreateWithFlags(&st[k], cudaStreamNonBlocking);
		if (!rc) rc = (int)cudaStreamWaitEvent(st[k], ready, 0);
		if (!rc) rc = (int)cudaHostAlloc((void **)&host[k], row * rows, cudaHostAllocDefault);
		if (!rc) rc = adc_scratch_alloc((void **)&dev[k], row * rows, st[k]);
	}
	// chunk c goes through buffer and stream c % 2: the host reads chunk c while chunk c - 1 is copied and reduced
	for (int c = 0, y0 = 0; y0 < H && !rc; c++, y0 += rows) {
		const int k = c & 1, n = std::min(rows, H - y0);
		rc = (int)cudaStreamSynchronize(st[k]);                       // chunk c - 2 has left host[k] and dev[k]
		if (!rc) rc = read_rows(f, D, H, W, y0, n, host[k]);
		if (!rc) rc = (int)cudaMemcpyAsync(dev[k], host[k], row * n, cudaMemcpyHostToDevice, st[k]);
		if (!rc) {
			const long hw = (long)n * W;
			volume_grey_kernel<<<(int)grid_for(hw), THREADS, 0, st[k]>>>(dev[k], D, hw, grey + (size_t)y0 * W);
			rc = (int)cudaPeekAtLastError();
		}
	}
	for (int k = 0; k < 2; k++) {
		if (!st[k]) continue;
		if (dev[k]) {
			const int r = adc_scratch_free(dev[k], st[k]);
			rc = rc ? rc : r;
		}
		const int r = (int)cudaStreamSynchronize(st[k]);
		rc = rc ? rc : r;
		cudaStreamDestroy(st[k]);
	}
	for (int k = 0; k < 2; k++)
		if (host[k]) cudaFreeHost(host[k]);
	if (ready) cudaEventDestroy(ready);
	fclose(f);
	return rc;
}

extern "C" int mccnn_render_map(const float *x, int H, int W, int d, unsigned char *grey, adcensus_stream_t stream)
{
	if (!x || !grey || H < 1 || W < 1 || d < 1 || (long)H * W >= (1l << 31)) return ADCENSUS_EINVAL;
	const long hw = (long)H * W;
	map_grey_kernel<<<(int)grid_for(hw), THREADS, 0, adc_stream(stream)>>>(x, hw, (float)d, grey);
	ADC_CHECK_LAUNCH();
	return 0;
}

extern "C" int mccnn_render_jet(const float *x, int H, int W, int disp_max, int mask_blue, unsigned char *rgb,
				adcensus_stream_t stream)
{
	if (!x || !rgb || H < 1 || W < 1 || disp_max < 1 || (long)H * W * 3 >= (1l << 31)) return ADCENSUS_EINVAL;
	cudaStream_t s = adc_stream(stream);
	const long hw = (long)H * W;
	int *flag = nullptr, refused = 0;
	int rc = adc_scratch_alloc((void **)&flag, sizeof(int), s);
	if (rc) return rc;
	rc = (int)cudaMemsetAsync(flag, 0, sizeof(int), s);
	if (!rc) {
		jet_kernel<<<(int)grid_for(hw), THREADS, 0, s>>>(x, hw, (double)disp_max, mask_blue, rgb, flag);
		rc = (int)cudaPeekAtLastError();
	}
	if (!rc) rc = (int)cudaMemcpyAsync(&refused, flag, sizeof(int), cudaMemcpyDeviceToHost, s);
	const int rf = adc_scratch_free(flag, s);
	if (!rc) rc = rf;
	if (!rc) rc = (int)cudaStreamSynchronize(s);
	return rc ? rc : (refused ? ADCENSUS_ERANGE : 0);
}

extern "C" int mccnn_render_error(const float *x0, const float *pred, const float *gt, int H, int W, float err_at,
				  unsigned char *rgb, adcensus_stream_t stream)
{
	if (!x0 || !pred || !gt || !rgb || H < 1 || W < 1 || !(err_at >= 0.f) || (long)H * W * 3 >= (1l << 31))
		return ADCENSUS_EINVAL;
	const long hw = (long)H * W;
	error_kernel<<<(int)grid_for(hw), THREADS, 0, adc_stream(stream)>>>(x0, pred, gt, hw, err_at, rgb);
	ADC_CHECK_LAUNCH();
	return 0;
}
