// pipeline.cu -- stereo_predict (main.lua:929-1082, arch 'fast') as one native
// object: every device buffer is allocated once at create time, a run is a fixed
// sequence of kernel launches (no allocation, no host sync) ordered on the caller's
// stream, so a batch driver can keep one pipeline per GPU / per stream busy back to
// back.  By default the two independent directions (main.lua:955) are overlapped:
// direction -1 runs on an internal side stream, started when direction +1 reaches
// its SGM phase, and the HBM-bound permute / SGM phases run on high-priority
// streams, so that they share the GPU with the issue-bound CBCA iterations of the
// other direction (mccnn_pipeline_set_overlap; joined before the LR check).
//
// Stage order, which volume is "left"/"right", the direction loop {+1,-1}, the /4
// and the permutes follow main.lua line by line (cited inline); the kernels are
// the ones behind the adcensus_* C ABI.
#include <initializer_list>
#include <math.h>
#include <new>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tma.cuh"

// internal entry points of the other translation units
size_t adc_packed_words(int H, int W);
int adc_pack_arms(const float *xc, uint32_t *pk, int which, int H, int W, int *maxlen_dev, cudaStream_t s);
int adc_cbca_packed(const uint32_t *pk, const float *x0c, const float *x1c,
		    const float *vol, float *out, int D, int H, int W, int ld, int direction, int maxlen, cudaStream_t s);
size_t adc_packed_hv_words(int H, int W);
int adc_pack_arms_hv(const float *xc, uint32_t *hv, int which, int H, int W, cudaStream_t s);
int adc_cbca_fast_pipeline_max_halo();
int adc_cbca_fast_box(int halo, int *box_w, int *box_h);
int adc_cbca_fast(const CUtensorMap *tm, const uint32_t *hv, const float *vol, float *out, int D, int H, int W, int ld, int direction,
		  int halo, cudaStream_t s);
size_t adc_sgm_table_bytes(int H, int W, int D);
int adc_sgm2_ckpt(const float *x0, const float *x1, const float *in, float *out, uint8_t *tab, void *scratch, size_t scratch_bytes,
		  int H, int W, int D, float pi1, float pi2, float tau_so, float alpha1, float q1, float q2, int direction, cudaStream_t s);
int adc_transpose_dhw_pitched_to_hwd(const float *in, float *out, int D, int H, int W, int ld, cudaStream_t s);
int adc_transpose_hwd_to_dhw_pitched_div4(const float *in, float *out, int D, int H, int W, int ld, cudaStream_t s);
int adc_stereo_join(const float *input_L, const float *input_R, float *output_L, float *output_R,
		    int C, int D, int H, int W, int ldo, cudaStream_t s);
int adc_fill_invalid(float *volL, float *volR, int D, int H, int W, int ld, cudaStream_t s);
int adc_fix_border(float *vol, int D, int H, int W, int ld, int n, int direction, cudaStream_t s);
int adc_argmin_pitched(const float *vol, float *disp, int D, int H, int W, int ld, cudaStream_t s);
int adc_argmin_conf_pitched(const float *vol, float *disp, float *conf, int D, int H, int W, int ld, cudaStream_t s);
int adc_subpixel(const float *d0, const float *c2, float *out, int H, int W, int ld, int disp_max, cudaStream_t s);

// Private volume layout: (D, H, ld), ld = W rounded up to a multiple of 4 floats.  Every row then starts on a
// 16-byte boundary: tensor maps (TMA) can describe the volumes, and 16-byte vector / cp.async accesses along x are
// legal everywhere (the API-facing (D,H,W) tensors with W = 1226 are only 8-byte aligned per row).  The padding
// columns hold unspecified values and are never read as data.
struct mccnn_pipeline {
	int C, D, H, W, ld, device;
	mccnn_params prm;
	long HW, V;       // H*W; elements of one private volume = D*H*ld
	size_t bytes;
	int launches;
	int cbca_mode;    // 1 = constant-work aggregation (default, 1e-4 contract), 0 = exact (bit-identical to the reference)
	size_t tab_bytes;
	// device buffers
	float *vols;      // 2V: [0] left volume, [1] right volume (main.lua:946)
	float *bufA;      // V : CBCA ping-pong
	float *bufC;      // V : SGM accumulator / ping-pong
	float *x0c, *x1c; // 4HW each: cross arms (main.lua:993-996)
	uint32_t *packed; // packed arm lengths of both images: bytes (exact kernels) + H/V words (constant-work kernel)
	int *maxlen;
	float *maps;      // 8HW: disparity maps and stage outputs
	float *gauss;     // ks*ks of the current blur_sigma, in a buffer of ks_alloc*ks_alloc floats
	uint8_t *sgmtab;  // SGM penalty-class tables
	int ks, ks_alloc;
	// tensor maps of the volume buffers (inputs of the TMA-staged CBCA), all encoded for the run shape
	// (tm_D, tm_H, tm_W); a run at another shape re-encodes them first (encode_maps), 0 = none valid
	int tm_D, tm_H, tm_W;
	int ntm;
	const float *tm_ptr[6];
	CUtensorMap tm[6];
	// direction overlap (mccnn_pipeline_set_overlap): the two directions of main.lua:955 are independent
	// until the LR check, so the second one runs on a side stream with its own ping-pong / SGM buffers,
	// started when the first reaches its SGM phase.
	int overlap;      // 0 off; otherwise two streams, the SGM phases on high-priority streams
	float *bufA2, *bufC2;
	uint8_t *sgmtab2;
	cudaStream_t side_stream, hi_stream[2];
	cudaEvent_t ev_stagger, ev_join, ev_hi_in[2], ev_hi_out[2];
	// staging for the host-buffer entry points: two slots so that the copy of pair i+1 overlaps
	// the kernels of pair i
	float *h_feat[2], *h_img[2], *h_disp[2];  // device copies per slot: 2F, 2HW, HW
	cudaStream_t own_stream, copy_stream, out_stream;
	cudaEvent_t ev_in[2], ev_free[2], ev_out[2];
	// further lanes of the batch entry points: a chain of twin pipelines (own buffers and streams) taking pairs round-robin, so that the
	// low-occupancy tail of one pair (LR check, interpolation, median, bilateral: many small kernels) and the bubbles
	// between its launches run next to the heavy kernels of the next pair
	mccnn_pipeline *twin;
	cudaEvent_t ev_fork, ev_lane;
};

extern "C" int mccnn_pipeline_set_overlap(mccnn_pipeline *p, int mode);

namespace {

int dev_alloc(void **p, size_t bytes, size_t *acc)
{
	cudaError_t e = cudaMalloc(p, bytes);
	if (e != cudaSuccess) return (int)e;
	*acc += bytes;
	return 0;
}

// longest arm cross() can produce for this preset, and the CBCA support radius
int pipe_maxlen(const mccnn_pipeline *p) { return p->prm.L1 > 2 ? p->prm.L1 : 2; }

// constant-work aggregation only for the arms the 1e-4 contract allows (cbca_tma.cu FAST_PIPELINE_MAX_HALO)
bool pipe_fast_cbca_ok(const mccnn_pipeline *p) { return pipe_maxlen(p) - 1 <= adc_cbca_fast_pipeline_max_halo(); }

// a map of `buf` as a (tm_D, tm_H, tm_W) volume with rows of tm_W rounded up to 4 floats
int add_tensor_map(mccnn_pipeline *p, const float *buf)
{
	if (!pipe_fast_cbca_ok(p)) return 0;               // such presets run the exact kernels
	const int halo = pipe_maxlen(p) - 1;
	if (!p->tm_D) return 0;                            // no valid shape: the next run encodes every map
	if (p->ntm >= 6) return ADCENSUS_EINVAL;
	int bw, bh;
	int rc = adc_cbca_fast_box(halo, &bw, &bh);
	if (!rc) rc = adc_tma_encode_volume(&p->tm[p->ntm], buf, p->tm_D, p->tm_H, p->tm_W, (p->tm_W + 3) & ~3, bw, bh);
	if (rc) return rc;
	p->tm_ptr[p->ntm++] = buf;
	return 0;
}

// (Re-)encode every tensor map for volumes of shape (D, H, W): the CBCA input maps of both volumes (the right one starts
// D*H*ld floats into `vols`), the ping-pong / accumulator buffers and, in overlap mode, the side stream's.  Kernels already
// launched are unaffected: each one received its map by value (__grid_constant__) at launch.
int encode_maps(mccnn_pipeline *p, int D, int H, int W)
{
	const int ld = (W + 3) & ~3;
	const long V = (long)D * H * ld;
	p->ntm = 0;
	p->tm_D = D; p->tm_H = H; p->tm_W = W;
	int rc = 0;
	for (const float *b : {(const float *)p->vols, (const float *)(p->vols + V), (const float *)p->bufA, (const float *)p->bufC,
			       (const float *)p->bufA2, (const float *)p->bufC2})
		if (!rc && b) rc = add_tensor_map(p, b);
	if (rc) {                                          // leave nothing half-encoded behind
		p->ntm = 0;
		p->tm_D = p->tm_H = p->tm_W = 0;
	}
	return rc;
}

const CUtensorMap *find_tensor_map(const mccnn_pipeline *p, const float *buf)
{
	for (int i = 0; i < p->ntm; i++)
		if (p->tm_ptr[i] == buf) return &p->tm[i];
	return nullptr;
}

struct DeviceGuard {
	int prev;
	explicit DeviceGuard(int dev) { cudaGetDevice(&prev); cudaSetDevice(dev); }
	~DeviceGuard() { cudaSetDevice(prev); }
};

bool terminate_ok(int c) { return c >= MCCNN_SM_NONE && c <= MCCNN_SM_MEDIAN; }
bool skip_ok(int c)
{
	return c == MCCNN_SM_NONE || c == MCCNN_SM_SGM || c == MCCNN_SM_OCCLUSION || c == MCCNN_SM_SUBPIXEL || c == MCCNN_SM_MEDIAN ||
	       c == MCCNN_SM_BILATERAL || c == MCCNN_SM_CBCA;
}

// the parameter checks shared by create and set_params; W = the created width
bool params_ok(const mccnn_params *o, int W)
{
	return o->cbca_i1 >= 0 && o->cbca_i2 >= 0 && o->sgm_i >= 0 && o->border >= 0 && o->border + 1 <= W &&
	       terminate_ok(o->sm_terminate) && skip_ok(o->sm_skip);
}

// Which steps of main.lua:953-1082 run under -sm_terminate / -sm_skip: sm_active starts true, a step runs while it is true
// and the step is not the skipped one, and passing the terminate step clears it.  The LR-check steps and their terminate
// names exist only for kitti (lr_check).
struct Stages {
	bool cbca1, sgm, cbca2, occlusion, mismatch, subpixel, median, bilateral;
};

Stages stages_of(const mccnn_params &o)
{
	const int T = o.sm_terminate, S = o.sm_skip;
	Stages st;
	bool active = T != MCCNN_SM_CNN;                                                          // :988
	st.cbca1 = active && S != MCCNN_SM_CBCA;                                                  // :992
	active = active && T != MCCNN_SM_CBCA1;                                                   // :1005
	st.sgm = active && S != MCCNN_SM_SGM;                                                     // :1007
	active = active && T != MCCNN_SM_SGM;                                                     // :1031
	st.cbca2 = active && S != MCCNN_SM_CBCA;                                                  // :1033
	active = active && T != MCCNN_SM_CBCA2;                                                   // :1040
	st.occlusion = o.lr_check && active && S != MCCNN_SM_OCCLUSION;                           // :1057
	if (o.lr_check) active = active && T != MCCNN_SM_OCCLUSION;                              // :1060
	st.mismatch = o.lr_check && active && S != MCCNN_SM_OCCLUSION;                            // :1062
	if (o.lr_check) active = active && T != MCCNN_SM_MISMATCH;                               // :1065
	st.subpixel = active && S != MCCNN_SM_SUBPIXEL;                                           // :1067
	active = active && T != MCCNN_SM_SUBPIXEL;                                                // :1071
	st.median = active && S != MCCNN_SM_MEDIAN;                                               // :1072
	active = active && T != MCCNN_SM_MEDIAN;                                                  // :1076
	st.bilateral = active && S != MCCNN_SM_BILATERAL;                                         // :1077
	return st;
}

// direction +1 is consumed only by the outlier map of the interpolations (or a caller that wants the right volume or the
// outlier map itself)
bool needs_right(const mccnn_params &o, const Stages &st, const float *volR, const float *lr)
{
	return (o.lr_check && (st.occlusion || st.mismatch)) || volR || lr;
}

// gaussian(blur_sigma) (main.lua:1078 gaussian(opt.blur_sigma):cuda()) into p->gauss; the buffer grows only when the kernel
// does not fit the one allocated.  Synchronous: the caller makes sure no enqueued run still reads the buffer.
int load_gauss(mccnn_pipeline *p, double sigma)
{
	const int ks = mccnn_gaussian(sigma, nullptr);
	const size_t f = sizeof(float);
	if (ks > p->ks_alloc) {
		if (p->gauss) {
			cudaFree(p->gauss);
			p->bytes -= (size_t)p->ks_alloc * p->ks_alloc * f;
			p->gauss = nullptr;
			p->ks_alloc = 0;
		}
		int rc = dev_alloc((void **)&p->gauss, (size_t)ks * ks * f, &p->bytes);
		if (rc) return rc;
		p->ks_alloc = ks;
	}
	float *hk = (float *)malloc((size_t)ks * ks * f);
	if (!hk) return ADCENSUS_EINVAL;
	mccnn_gaussian(sigma, hk);
	int rc = (int)cudaMemcpy(p->gauss, hk, (size_t)ks * ks * f, cudaMemcpyHostToDevice);
	free(hk);
	if (!rc) p->ks = ks;
	return rc;
}

}  // namespace

extern "C" int mccnn_pipeline_create(mccnn_pipeline **out, int C, int D, int H, int W, const mccnn_params *params, int device)
{
	if (!out || !params || C < 1 || D < 1 || H < 1 || W < 1) return ADCENSUS_EINVAL;
	if (C > 128 || D > ADCENSUS_MAX_DISP) return ADCENSUS_ELIMIT;
	if (!params_ok(params, W)) return ADCENSUS_EINVAL;
	DeviceGuard g(device);
	mccnn_pipeline *p = new (std::nothrow) mccnn_pipeline();
	if (!p) return ADCENSUS_EINVAL;
	memset(p, 0, sizeof(*p));
	p->C = C; p->D = D; p->H = H; p->W = W; p->device = device;
	p->ld = (W + 3) & ~3;
	p->prm = *params;
	p->HW = (long)H * W;
	p->V = (long)D * H * p->ld;
	const char *ex = getenv("ADCENSUS_CBCA_EXACT");
	p->cbca_mode = (ex && atoi(ex)) ? 0 : 1;
	p->tab_bytes = adc_sgm_table_bytes(H, W, D);
	int rc = 0;
	const size_t f = sizeof(float);
	if (!rc) rc = dev_alloc((void **)&p->vols, 2 * p->V * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->bufA, p->V * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->bufC, p->V * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->x0c, 4 * p->HW * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->x1c, 4 * p->HW * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->packed, (adc_packed_words(H, W) + adc_packed_hv_words(H, W)) * sizeof(uint32_t), &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->maxlen, sizeof(int), &p->bytes);
	if (!rc) rc = (int)cudaMemset(p->maxlen, 0, sizeof(int));
	if (!rc) rc = dev_alloc((void **)&p->maps, 8 * p->HW * f, &p->bytes);
	if (!rc) rc = dev_alloc((void **)&p->sgmtab, p->tab_bytes, &p->bytes);
	if (!rc) rc = encode_maps(p, D, H, W);
	if (!rc) rc = load_gauss(p, params->blur_sigma);
	if (rc) {
		mccnn_pipeline_destroy(p);
		return rc;
	}
	*out = p;
	// Default schedule: the two directions overlapped, 6V of volume buffers instead of 4V; if the extra buffers do not
	// fit, the sequential schedule is kept (same results).
	mccnn_pipeline_set_overlap(p, 2);
	return 0;
}

static void overlap_release(mccnn_pipeline *p);

extern "C" void mccnn_pipeline_destroy(mccnn_pipeline *p)
{
	if (!p) return;
	DeviceGuard g(p->device);
	cudaFree(p->vols); cudaFree(p->bufA); cudaFree(p->bufC); cudaFree(p->x0c); cudaFree(p->x1c);
	cudaFree(p->packed); cudaFree(p->maxlen); cudaFree(p->maps); cudaFree(p->gauss); cudaFree(p->sgmtab);
	for (int k = 0; k < 2; k++) {
		cudaFree(p->h_feat[k]); cudaFree(p->h_img[k]); cudaFree(p->h_disp[k]);
		if (p->ev_in[k]) cudaEventDestroy(p->ev_in[k]);
		if (p->ev_free[k]) cudaEventDestroy(p->ev_free[k]);
		if (p->ev_out[k]) cudaEventDestroy(p->ev_out[k]);
	}
	overlap_release(p);
	if (p->twin) mccnn_pipeline_destroy(p->twin);
	if (p->ev_fork) cudaEventDestroy(p->ev_fork);
	if (p->ev_lane) cudaEventDestroy(p->ev_lane);
	if (p->own_stream) cudaStreamDestroy(p->own_stream);
	if (p->copy_stream) cudaStreamDestroy(p->copy_stream);
	if (p->out_stream) cudaStreamDestroy(p->out_stream);
	delete p;
}

extern "C" size_t mccnn_pipeline_device_bytes(const mccnn_pipeline *p) { return p ? p->bytes : 0; }
// 1 (default) constant-work aggregation within the 1e-4 contract (cbca_tma.cu); 0 exact, bit-identical to the reference
extern "C" void mccnn_pipeline_set_cbca_mode(mccnn_pipeline *p, int mode) { if (p) p->cbca_mode = mode ? 1 : 0; }
extern "C" int mccnn_pipeline_get_cbca_mode(const mccnn_pipeline *p) { return p ? p->cbca_mode : -1; }
static void overlap_release(mccnn_pipeline *p)
{
	const size_t f = sizeof(float);
	if (p->bufA2) { cudaFree(p->bufA2); p->bytes -= p->V * f; }
	if (p->bufC2) { cudaFree(p->bufC2); p->bytes -= p->V * f; }
	if (p->sgmtab2) { cudaFree(p->sgmtab2); p->bytes -= p->tab_bytes; }
	for (int i = 0; i < p->ntm;)                       // forget the maps of the released buffers
		if (p->tm_ptr[i] == p->bufA2 || p->tm_ptr[i] == p->bufC2) {
			p->tm_ptr[i] = p->tm_ptr[p->ntm - 1];
			p->tm[i] = p->tm[p->ntm - 1];
			p->ntm--;
		} else {
			i++;
		}
	p->bufA2 = p->bufC2 = nullptr;
	p->sgmtab2 = nullptr;
	if (p->side_stream) cudaStreamDestroy(p->side_stream);
	if (p->ev_stagger) cudaEventDestroy(p->ev_stagger);
	if (p->ev_join) cudaEventDestroy(p->ev_join);
	p->side_stream = nullptr; p->ev_stagger = nullptr; p->ev_join = nullptr;
	for (int k = 0; k < 2; k++) {
		if (p->hi_stream[k]) cudaStreamDestroy(p->hi_stream[k]);
		if (p->ev_hi_in[k]) cudaEventDestroy(p->ev_hi_in[k]);
		if (p->ev_hi_out[k]) cudaEventDestroy(p->ev_hi_out[k]);
		p->hi_stream[k] = nullptr; p->ev_hi_in[k] = nullptr; p->ev_hi_out[k] = nullptr;
	}
	p->overlap = 0;
}

extern "C" int mccnn_pipeline_set_overlap(mccnn_pipeline *p, int mode)
{
	if (!p || mode < 0 || mode > 2) return ADCENSUS_EINVAL;
	DeviceGuard g(p->device);
	if (mode && !p->side_stream) {
		const size_t f = sizeof(float);
		int rc = 0, lo = 0, hi = 0;
		if (!rc) rc = dev_alloc((void **)&p->bufA2, p->V * f, &p->bytes);
		if (!rc) rc = dev_alloc((void **)&p->bufC2, p->V * f, &p->bytes);
		if (!rc) rc = dev_alloc((void **)&p->sgmtab2, p->tab_bytes, &p->bytes);
		if (!rc) rc = add_tensor_map(p, p->bufA2);
		if (!rc) rc = add_tensor_map(p, p->bufC2);
		if (!rc) rc = (int)cudaDeviceGetStreamPriorityRange(&lo, &hi);   // hi = numerically lowest = greatest priority
		if (!rc) rc = (int)cudaStreamCreateWithPriority(&p->side_stream, cudaStreamNonBlocking, lo);
		for (int k = 0; k < 2 && !rc; k++) {
			rc = (int)cudaStreamCreateWithPriority(&p->hi_stream[k], cudaStreamNonBlocking, hi);
			if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_hi_in[k], cudaEventDisableTiming);
			if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_hi_out[k], cudaEventDisableTiming);
		}
		if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_stagger, cudaEventDisableTiming);
		if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming);
		if (rc) {                                      // leave the pipeline as it was (sequential mode still works)
			overlap_release(p);
			cudaGetLastError();
			return rc;
		}
	}
	p->overlap = mode;
	return 0;
}

extern "C" int mccnn_pipeline_launches_per_run(const mccnn_pipeline *p) { return p ? p->launches : 0; }

// Re-targets the pipeline (and every twin lane) to another parameter set.  What create derived from the parameters is
// derived again: the Gaussian (main.lua:1078) and the tensor maps, whose box and very existence depend on the arm bound
// max(L1, 2) -- the maps are dropped here and the next run encodes them for its shape, as after a shape change.
extern "C" int mccnn_pipeline_set_params(mccnn_pipeline *p, const mccnn_params *params)
{
	if (!p || !params || !params_ok(params, p->W)) return ADCENSUS_EINVAL;
	DeviceGuard g(p->device);
	ADC_CUDA(cudaDeviceSynchronize());                 // enqueued runs read the Gaussian and the parameters' kernel choice
	for (mccnn_pipeline *q = p; q; q = q->twin) {
		int rc = load_gauss(q, params->blur_sigma);
		if (rc) return rc;
		q->prm = *params;
		q->ntm = 0;
		q->tm_D = q->tm_H = q->tm_W = 0;
	}
	return 0;
}

#define STEP(call)                 \
	do {                       \
		int rc__ = (call); \
		if (rc__) return rc__; \
	} while (0)

// A run at (H, W, D) <= the created shape: every shape-dependent quantity (row pitch, volume size, the offset of the
// right volume, map offsets, table sizes, tensor maps) is derived from the run shape, so the buffers hold exactly
// what a pipeline created at this shape would hold.  run_fits checks the shape against the allocations and encodes the
// tensor maps for it; then the volumes are built (run_build_volumes) or copied in (mccnn_pipeline_run_volumes), and
// run_chain takes them from cross/CBCA to the disparity map.
static int run_fits(mccnn_pipeline *p, int H, int W, int D)
{
	const int ld = (W + 3) & ~3;
	const long HW = (long)H * W, V = (long)D * H * ld;
	// the allocations were sized for the created shape; check the run's needs against them instead of assuming
	if (V > p->V || HW > p->HW) return ADCENSUS_ELIMIT;
	if (adc_packed_words(H, W) + adc_packed_hv_words(H, W) > adc_packed_words(p->H, p->W) + adc_packed_hv_words(p->H, p->W))
		return ADCENSUS_ELIMIT;
	if (adc_sgm_table_bytes(H, W, D) > p->tab_bytes) return ADCENSUS_ELIMIT;
	if (p->tm_D != D || p->tm_H != H || p->tm_W != W) STEP(encode_maps(p, D, H, W));
	return 0;
}

// main.lua:946-949: both cost volumes of the pair into the private pitched buffers; returns the number of kernel launches
static int run_build_volumes(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR, cudaStream_t s,
			     int *launches)
{
	const int C = p->C, ld = (W + 3) & ~3;
	const long V = (long)D * H * ld;
	const mccnn_params &o = p->prm;
	int nl = 0;
	float *volsL = p->vols, *volsR = p->vols + V;
	STEP(adc_fill_invalid(volsL, volsR, D, H, W, ld, s)); nl += 1;                                 // main.lua:946 (only what :947 leaves)
	STEP(adc_stereo_join(featL, featR, volsL, volsR, C, D, H, W, ld, s)); nl += 1;                  // :947
	STEP(adc_fix_border(volsL, D, H, W, ld, o.border, -1, s));                                    // :948
	STEP(adc_fix_border(volsR, D, H, W, ld, o.border, 1, s)); nl += o.border ? 2 : 0;             // :949
	*launches = nl;
	return 0;
}

// main.lua:986-1082 from the two volumes in the private buffers (the right one only when it is consumed); nl = the
// launches that built them.  conf: the margin confidence of the final left volume, from direction -1's arg-min (same
// launch count); lr: main.lua:1056's outlier map, for which direction +1 and the LR check run if nothing else needs them.
static int run_chain(mccnn_pipeline *p, int H, int W, int D, const float *imgL, const float *imgR, float *disp, float *volL,
		     float *volR, float *conf, float *lr, int nl, cudaStream_t s)
{
	const int ld = (W + 3) & ~3;
	const long HW = (long)H * W, V = (long)D * H * ld;
	const mccnn_params &o = p->prm;
	const Stages st = stages_of(o);
	float *volsL = p->vols, *volsR = p->vols + V;
	const int cbca_i1 = st.cbca1 ? o.cbca_i1 : 0, cbca_i2 = st.cbca2 ? o.cbca_i2 : 0, sgm_i = st.sgm ? o.sgm_i : 0;

	// cross arms: identical for both directions (main.lua:993-996 recomputes them)
	const int maxlen = pipe_maxlen(p);       // bound on the arm length cross() can produce
	const int ncbca = cbca_i1 + cbca_i2;
	// fix_border copies column W-n-1 over the border columns: for D > W - n - 1 that column holds NaN at "valid"
	// positions, which only the tap-by-tap generic kernel treats like the reference (NaN only where a tap is NaN)
	const bool nan_in_valid = o.border > 0 && D > W - o.border - 1;
	const bool tma = p->cbca_mode && !nan_in_valid && pipe_fast_cbca_ok(p) && p->ntm > 0;
	uint32_t *hv = p->packed + adc_packed_words(H, W);
	if (ncbca > 0) {
		STEP(adcensus_cross(imgL, p->x0c, H, W, o.L1, o.tau1, s));
		STEP(adcensus_cross(imgR, p->x1c, H, W, o.L1, o.tau1, s)); nl += 2;
		if (tma) {
			STEP(adc_pack_arms_hv(p->x0c, hv, 0, H, W, s));
			STEP(adc_pack_arms_hv(p->x1c, hv, 1, H, W, s)); nl += 2;
		} else if (!nan_in_valid) {
			STEP(adc_pack_arms(p->x0c, p->packed, 0, H, W, p->maxlen, s));
			STEP(adc_pack_arms(p->x1c, p->packed, 1, H, W, p->maxlen, s)); nl += 2;
		}
	}
	auto cbca = [&](const float *in, float *out, int direction, cudaStream_t ds) -> int {        // adcensus.cbca, :999 / :1036
		if (tma) {
			const CUtensorMap *tm = find_tensor_map(p, in);
			if (!tm) return ADCENSUS_EINVAL;
			return adc_cbca_fast(tm, hv, in, out, D, H, W, ld, direction, maxlen - 1, ds);
		}
		return adc_cbca_packed(p->packed, p->x0c, p->x1c, in, out, D, H, W, ld, direction, nan_in_valid ? (1 << 20) : maxlen, ds);
	};

	// every map is written straight into `disp` when no later step runs (an early -sm_terminate, or skipped tail steps)
	const bool after_mis = st.subpixel || st.median || st.bilateral, after_occ = st.mismatch || after_mis;
	float *m = p->maps;
	float *dispR = m, *dispL = (st.occlusion || after_occ) ? m + HW : disp;
	float *final_left = nullptr;
	// One direction of main.lua:955-1051 on stream `ds`: cur/spare ping-pong, acc = SGM accumulator.
	// k = 0: direction +1 (right volume), k = 1: direction -1 (left volume).
	auto run_direction = [&](int k, cudaStream_t ds, float *cur, float *spare, float *acc, uint8_t *tab) -> int {
		const int direction = k == 0 ? 1 : -1;                                                   // :955
		for (int i = 0; i < cbca_i1; i++) {                                                      // :998-1001
			STEP(cbca(cur, spare, direction, ds));
			float *t = cur; cur = spare; spare = t; nl += 1;
		}
		if (k == 0 && p->overlap) STEP((int)cudaEventRecord(p->ev_stagger, ds));                 // the other direction may start
		cudaStream_t ss = ds;                                                                    // stream of the SGM phase
		if (p->overlap && sgm_i > 0) {
			ss = p->hi_stream[k];
			STEP((int)cudaEventRecord(p->ev_hi_in[k], ds));
			STEP((int)cudaStreamWaitEvent(ss, p->ev_hi_in[k], 0));
		}
		for (int it = 0; it < sgm_i; it++) {                                                     // :1008-1020
			STEP(adc_transpose_dhw_pitched_to_hwd(cur, spare, D, H, W, ld, ss));                 // :1008
			// cur is dead between the two transposes: it holds SGM's line-state checkpoints
			STEP(adc_sgm2_ckpt(imgL, imgR, spare, acc, tab, cur, (size_t)V * sizeof(float), H, W, D, o.pi1, o.pi2,
					   o.tau_so, o.alpha1, o.sgm_q1, o.sgm_q2, direction, ss));                // :1014-1016
			STEP(adc_transpose_hwd_to_dhw_pitched_div4(acc, cur, D, H, W, ld, ss));              // :1017-1020
			nl += 7;
		}
		if (ss != ds) {
			STEP((int)cudaEventRecord(p->ev_hi_out[k], ss));
			STEP((int)cudaStreamWaitEvent(ds, p->ev_hi_out[k], 0));
		}
		for (int i = 0; i < cbca_i2; i++) {                                                      // :1035-1038
			STEP(cbca(cur, spare, direction, ds));
			float *t = cur; cur = spare; spare = t; nl += 1;
		}
		if (direction == -1 && conf)                                                             // :1049-1050
			STEP(adc_argmin_conf_pitched(cur, dispL, conf, D, H, W, ld, ds));
		else
			STEP(adc_argmin_pitched(cur, direction == 1 ? dispR : dispL, D, H, W, ld, ds));
		nl += 1;
		float *dst = direction == 1 ? volR : volL;                                               // :1042-1047
		if (dst) STEP((int)cudaMemcpy2DAsync(dst, (size_t)W * 4, cur, (size_t)ld * 4, (size_t)W * 4, (size_t)D * H,
						     cudaMemcpyDeviceToDevice, ds));
		if (direction == -1) final_left = cur;
		return 0;
	};
	// main.lua:954-955: without the LR check (mb) only direction -1 is consumed, unless the caller asks for the
	// right volume (`-a predict` writes right.bin); with it, only when an interpolation reads the outlier map
	const bool need_right = needs_right(o, st, volR, lr);
	if (!need_right) {
		STEP(run_direction(1, s, volsL, p->bufA, p->bufC, p->sgmtab));
	} else if (!p->overlap) {
		// sequential: the right direction's three buffers are dead after its argmin / copy-out
		STEP(run_direction(0, s, volsR, p->bufA, p->bufC, p->sgmtab));
		STEP(run_direction(1, s, volsL, p->bufA, p->bufC, p->sgmtab));
	} else {
		// concurrent: direction -1 on the side stream with its own spare / accumulator / tables,
		// started when direction +1 leaves its first CBCA block
		STEP(run_direction(0, s, volsR, p->bufA, p->bufC, p->sgmtab));
		STEP((int)cudaStreamWaitEvent(p->side_stream, p->ev_stagger, 0));
		STEP(run_direction(1, p->side_stream, volsL, p->bufA2, p->bufC2, p->sgmtab2));
		STEP((int)cudaEventRecord(p->ev_join, p->side_stream));
		STEP((int)cudaStreamWaitEvent(s, p->ev_join, 0));
	}

	const float *curd = dispL;                                                                   // disp[2]
	float *outlier = lr ? lr : m + 2 * HW;
	if (st.occlusion || st.mismatch || lr) {                                                     // :1056 (unread otherwise)
		STEP(adcensus_outlier_detection(dispL, dispR, outlier, H, W, D, s)); nl += 1;
	}
	if (st.occlusion) {                                                                          // :1058
		float *out = after_occ ? m + 3 * HW : disp;
		STEP(adcensus_interpolate_occlusion(curd, outlier, out, H, W, s)); nl += 1;
		curd = out;
	}
	if (st.mismatch) {                                                                           // :1063
		float *out = after_mis ? m + 4 * HW : disp;
		STEP(adcensus_interpolate_mismatch(curd, outlier, out, H, W, s)); nl += 1;
		curd = out;
	}
	if (st.subpixel) {                                                                           // :1068
		float *out = st.median || st.bilateral ? m + 5 * HW : disp;
		STEP(adc_subpixel(curd, final_left, out, H, W, ld, D, s)); nl += 1;
		curd = out;
	}
	if (st.median) {                                                                             // :1073
		float *out = st.bilateral ? m + 6 * HW : disp;
		STEP(adcensus_median2d(curd, out, H, W, 5, s)); nl += 1;
		curd = out;
	}
	if (st.bilateral) {                                                                          // :1078
		STEP(adcensus_mean2d(curd, p->gauss, disp, H, W, p->ks, o.blur_t, s)); nl += 1;
	}
	p->launches = nl;
	return 0;
}

static int pipeline_run_at(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR,
			   const float *imgL, const float *imgR, float *disp, float *volL, float *volR, float *conf, float *lr,
			   cudaStream_t s)
{
	int nl = 0;
	STEP(run_fits(p, H, W, D));
	STEP(run_build_volumes(p, H, W, D, featL, featR, s, &nl));
	return run_chain(p, H, W, D, imgL, imgR, disp, volL, volR, conf, lr, nl, s);
}

extern "C" int mccnn_pipeline_run_volumes_conf(mccnn_pipeline *p, int H, int W, int D, const float *volL, const float *volR,
					       const float *imgL, const float *imgR, float *disp, float *conf, float *lr, float *outL,
					       float *outR, adcensus_stream_t stream)
{
	if (!p || !volL || !imgL || !imgR || !disp) return ADCENSUS_EINVAL;
	if (lr && !p->prm.lr_check) return ADCENSUS_EINVAL;                    // main.lua has no LR check there
	if (!volR && (p->prm.lr_check || outR)) return ADCENSUS_EINVAL;       // direction +1 is run: it needs its volume
	if (H < 1 || W < 1 || D < 1 || p->prm.border + 1 > W) return ADCENSUS_EINVAL;
	if (H > p->H || W > p->W || D > p->D) return ADCENSUS_ELIMIT;
	DeviceGuard g(p->device);
	cudaStream_t s = adc_stream(stream);
	STEP(run_fits(p, H, W, D));
	const int ld = (W + 3) & ~3;
	const long V = (long)D * H * ld;
	const size_t row = (size_t)W * sizeof(float), pitch = (size_t)ld * sizeof(float);
	ADC_CUDA(cudaMemcpy2DAsync(p->vols, pitch, volL, row, row, (size_t)D * H, cudaMemcpyDeviceToDevice, s));
	if (needs_right(p->prm, stages_of(p->prm), outR, lr))                  // only then is the right volume read
		ADC_CUDA(cudaMemcpy2DAsync(p->vols + V, pitch, volR, row, row, (size_t)D * H, cudaMemcpyDeviceToDevice, s));
	return run_chain(p, H, W, D, imgL, imgR, disp, outL, outR, conf, lr, 0, s);
}

extern "C" int mccnn_pipeline_run_volumes(mccnn_pipeline *p, int H, int W, int D, const float *volL, const float *volR,
					  const float *imgL, const float *imgR, float *disp, float *outL, float *outR,
					  adcensus_stream_t stream)
{
	return mccnn_pipeline_run_volumes_conf(p, H, W, D, volL, volR, imgL, imgR, disp, nullptr, nullptr, outL, outR, stream);
}

extern "C" int mccnn_pipeline_run(mccnn_pipeline *p, const float *featL, const float *featR,
				  const float *imgL, const float *imgR, float *disp,
				  float *volL, float *volR, adcensus_stream_t stream)
{
	if (!p || !featL || !featR || !imgL || !imgR || !disp) return ADCENSUS_EINVAL;
	DeviceGuard g(p->device);
	return pipeline_run_at(p, p->H, p->W, p->D, featL, featR, imgL, imgR, disp, volL, volR, nullptr, nullptr, adc_stream(stream));
}

extern "C" int mccnn_pipeline_run_shape_conf(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR,
					     const float *imgL, const float *imgR, float *disp, float *conf, float *lr, float *volL,
					     float *volR, adcensus_stream_t stream)
{
	if (!p || !featL || !featR || !imgL || !imgR || !disp) return ADCENSUS_EINVAL;
	if (lr && !p->prm.lr_check) return ADCENSUS_EINVAL;
	if (H < 1 || W < 1 || D < 1 || p->prm.border + 1 > W) return ADCENSUS_EINVAL;
	if (H > p->H || W > p->W || D > p->D) return ADCENSUS_ELIMIT;
	DeviceGuard g(p->device);
	return pipeline_run_at(p, H, W, D, featL, featR, imgL, imgR, disp, volL, volR, conf, lr, adc_stream(stream));
}

extern "C" int mccnn_pipeline_run_shape(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR,
					const float *imgL, const float *imgR, float *disp, float *volL, float *volR,
					adcensus_stream_t stream)
{
	return mccnn_pipeline_run_shape_conf(p, H, W, D, featL, featR, imgL, imgR, disp, nullptr, nullptr, volL, volR, stream);
}

static int host_staging(mccnn_pipeline *p)
{
	if (p->own_stream) return 0;
	const size_t F = (size_t)p->C * p->HW * sizeof(float), I = (size_t)p->HW * sizeof(float);
	int rc = 0;
	for (int k = 0; k < 2 && !rc; k++) {
		if (!rc) rc = dev_alloc((void **)&p->h_feat[k], 2 * F, &p->bytes);
		if (!rc) rc = dev_alloc((void **)&p->h_img[k], 2 * I, &p->bytes);
		if (!rc) rc = dev_alloc((void **)&p->h_disp[k], I, &p->bytes);
		if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_in[k], cudaEventDisableTiming);
		if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_free[k], cudaEventDisableTiming);
		if (!rc) rc = (int)cudaEventCreateWithFlags(&p->ev_out[k], cudaEventDisableTiming);
	}
	if (!rc) rc = (int)cudaStreamCreateWithFlags(&p->copy_stream, cudaStreamNonBlocking);
	if (!rc) rc = (int)cudaStreamCreateWithFlags(&p->out_stream, cudaStreamNonBlocking);
	if (!rc) rc = (int)cudaStreamCreateWithFlags(&p->own_stream, cudaStreamNonBlocking);
	return rc;
}

// the extra lanes (see struct): a chain of twins created on first use with the same parameters and modes; lane 0 is the
// pipeline itself.
static const int BATCH_LANES = 2;
static int batch_lanes(mccnn_pipeline *p, mccnn_pipeline **lane, int want)
{
	const int nl = want < BATCH_LANES ? want : BATCH_LANES;
	lane[0] = p;
	int n = 1;
	for (mccnn_pipeline *q = p; n < nl; n++) {
		if (!q->twin) {
			mccnn_pipeline *t = nullptr;
			if (mccnn_pipeline_create(&t, p->C, p->D, p->H, p->W, &p->prm, p->device)) {
				cudaGetLastError();
				break;                                 // not enough memory for another lane: fewer lanes give the same results
			}
			q->twin = t;
		}
		q = q->twin;
		q->cbca_mode = p->cbca_mode;
		if (q->overlap != p->overlap) mccnn_pipeline_set_overlap(q, p->overlap);
		lane[n] = q;
	}
	return n;
}

// pair number j of lane q from host memory: inputs are copied on q's copy stream into staging slot j % 2 while the lane's
// previous pair computes; the disparity map goes back on q's output stream
// cs: the H2D stream SHARED by the lanes (copies of different lanes would otherwise split the PCIe bandwidth and both arrive late:
// in order, pair i lands one transfer time after pair i - 1)
static int enqueue_host_pair(mccnn_pipeline *q, int j, cudaStream_t cs, const float *featL, const float *featR, const float *imgL, const float *imgR, float *disp)
{
	const size_t F = (size_t)q->C * q->HW * sizeof(float), I = (size_t)q->HW * sizeof(float);
	cudaStream_t ks = q->own_stream, os = q->out_stream;  // kernels, D2H
	const int k = j & 1;
	float *fL = q->h_feat[k], *fR = fL + (size_t)q->C * q->HW;
	float *iL = q->h_img[k], *iR = iL + q->HW;
	if (j >= 2) ADC_CUDA(cudaStreamWaitEvent(cs, q->ev_free[k], 0));   // slot's previous pair consumed
	ADC_CUDA(cudaMemcpyAsync(fL, featL, F, cudaMemcpyHostToDevice, cs));
	ADC_CUDA(cudaMemcpyAsync(fR, featR, F, cudaMemcpyHostToDevice, cs));
	ADC_CUDA(cudaMemcpyAsync(iL, imgL, I, cudaMemcpyHostToDevice, cs));
	ADC_CUDA(cudaMemcpyAsync(iR, imgR, I, cudaMemcpyHostToDevice, cs));
	ADC_CUDA(cudaEventRecord(q->ev_in[k], cs));
	ADC_CUDA(cudaStreamWaitEvent(ks, q->ev_in[k], 0));
	if (j >= 2) ADC_CUDA(cudaStreamWaitEvent(ks, q->ev_out[k], 0));     // slot's previous result copied out
	STEP(mccnn_pipeline_run(q, fL, fR, iL, iR, q->h_disp[k], nullptr, nullptr, ks));
	ADC_CUDA(cudaEventRecord(q->ev_free[k], ks));
	ADC_CUDA(cudaStreamWaitEvent(os, q->ev_free[k], 0));
	ADC_CUDA(cudaMemcpyAsync(disp, q->h_disp[k], I, cudaMemcpyDeviceToHost, os));
	ADC_CUDA(cudaEventRecord(q->ev_out[k], os));
	return 0;
}

// n pairs from host memory (pinned for real overlap): separate H2D / kernel / D2H streams with two staging slots per lane,
// pairs round-robin over the lanes (buffer sets, see batch_lanes).  Returns when every result is in its host buffer.
extern "C" int mccnn_pipeline_run_host_batch(mccnn_pipeline *p, int n, const float *const *featL_host,
					     const float *const *featR_host, const float *const *imgL_host,
					     const float *const *imgR_host, float *const *disp_host)
{
	if (!p || n < 0 || (n > 0 && (!featL_host || !featR_host || !imgL_host || !imgR_host || !disp_host))) return ADCENSUS_EINVAL;
	for (int i = 0; i < n; i++)
		if (!featL_host[i] || !featR_host[i] || !imgL_host[i] || !imgR_host[i] || !disp_host[i]) return ADCENSUS_EINVAL;
	DeviceGuard g(p->device);
	mccnn_pipeline *lane[BATCH_LANES];
	const int nl = batch_lanes(p, lane, n > 1 ? n : 1);
	for (int l = 0; l < nl; l++) STEP(host_staging(lane[l]));
	for (int i = 0; i < n; i++)
		STEP(enqueue_host_pair(lane[i % nl], i / nl, p->copy_stream, featL_host[i], featR_host[i], imgL_host[i], imgR_host[i], disp_host[i]));
	for (int l = 0; l < nl; l++) {
		ADC_CUDA(cudaStreamSynchronize(lane[l]->out_stream));
		ADC_CUDA(cudaStreamSynchronize(lane[l]->own_stream));
		ADC_CUDA(cudaStreamSynchronize(lane[l]->copy_stream));
	}
	return 0;
}

// n device-resident pairs, ordered on `stream` as a whole (everything enqueued before the call precedes it, everything after
// it sees all n disparity maps): pairs alternate between the two lanes on their own streams.
extern "C" int mccnn_pipeline_run_batch(mccnn_pipeline *p, int n, const float *const *featL, const float *const *featR,
					const float *const *imgL, const float *const *imgR, float *const *disp, adcensus_stream_t stream)
{
	if (!p || n < 0 || (n > 0 && (!featL || !featR || !imgL || !imgR || !disp))) return ADCENSUS_EINVAL;
	for (int i = 0; i < n; i++)
		if (!featL[i] || !featR[i] || !imgL[i] || !imgR[i] || !disp[i]) return ADCENSUS_EINVAL;
	DeviceGuard g(p->device);
	cudaStream_t s = adc_stream(stream);
	mccnn_pipeline *lane[BATCH_LANES];
	const int nl = batch_lanes(p, lane, n > 1 ? n : 1);
	if (nl == 1) {
		for (int i = 0; i < n; i++) STEP(mccnn_pipeline_run(p, featL[i], featR[i], imgL[i], imgR[i], disp[i], nullptr, nullptr, s));
		return 0;
	}
	for (int l = 0; l < nl; l++) {
		STEP(host_staging(lane[l]));                        // creates the lanes' own streams
		if (!lane[l]->ev_lane) ADC_CUDA(cudaEventCreateWithFlags(&lane[l]->ev_lane, cudaEventDisableTiming));
	}
	if (!p->ev_fork) ADC_CUDA(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
	ADC_CUDA(cudaEventRecord(p->ev_fork, s));
	for (int l = 0; l < nl; l++) ADC_CUDA(cudaStreamWaitEvent(lane[l]->own_stream, p->ev_fork, 0));
	for (int i = 0; i < n; i++) {
		mccnn_pipeline *q = lane[i % nl];
		STEP(mccnn_pipeline_run(q, featL[i], featR[i], imgL[i], imgR[i], disp[i], nullptr, nullptr, q->own_stream));
	}
	for (int l = 0; l < nl; l++) {
		ADC_CUDA(cudaEventRecord(lane[l]->ev_lane, lane[l]->own_stream));
		ADC_CUDA(cudaStreamWaitEvent(s, lane[l]->ev_lane, 0));
	}
	return 0;
}

extern "C" int mccnn_pipeline_run_host(mccnn_pipeline *p, const float *featL_host, const float *featR_host,
				       const float *imgL_host, const float *imgR_host, float *disp_host)
{
	return mccnn_pipeline_run_host_batch(p, 1, &featL_host, &featR_host, &imgL_host, &imgR_host, &disp_host);
}
