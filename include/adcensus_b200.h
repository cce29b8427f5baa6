/*
 * adcensus_b200.h -- C ABI of libadcensus_b200.so, the H100 (sm_90a) drop-in
 * for the stereo-method hot path of jzbontar/mc-cnn's libadcensus.so.
 *
 * The reference exposes this path only as lua_CFunctions registered into the
 * Lua table `adcensus` (adcensus.cu:2061-2105).  Each `adcensus_<name>` below
 * is the plain-C core that the Lua face (csrc/lua_face.cu,
 * luaopen_libadcensus) -- or any other FFI: cgo, ctypes, JNI -- binds for the
 * Lua function of the same name; arguments are the tensors' raw device
 * pointers plus the sizes the reference reads from the tensors themselves.
 * See INTEGRATION.md for the binding a maintainer adds.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous float32 (the reference
 *     ignores strides: raw THCudaTensor_data + sizes);
 *   - shapes: features (C,H,W); cost volumes (D,H,W); SGM volumes (H,W,D); `*_pitched` entry points take
 *     (D,H,ld) volumes with a row pitch ld (the fused pipeline's private layout);
 *     images / disparity maps (H,W); cross arms (4,H,W);
 *   - `stream` is a cudaStream_t (0 = legacy default stream, what the
 *     reference launches on); all work is asynchronous on it unless noted;
 *   - return 0 on success, a positive cudaError_t, or a negative ADCENSUS_E*
 *     for arguments the kernels cannot handle (the reference's compiled-out
 *     device asserts: C <= 128 adcensus.cu:1460, D <= 400 :574, H <= W for
 *     sgm2's tmp :570).  Nothing here ever falls back to a CPU path.
 *   - no function keeps a pointer after it returns; the library holds no
 *     global mutable state apart from a per-device scratch pool that is
 *     stream-ordered (cudaMallocAsync).
 */
#ifndef ADCENSUS_B200_H
#define ADCENSUS_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ADCENSUS_EINVAL (-1)   /* bad size / null pointer / unsupported value */
#define ADCENSUS_ELIMIT (-2)   /* exceeds a documented limit (D, C, ksize ...) */

#define ADCENSUS_MAX_DISP 512      /* sgm2: reference tree-min covers d < 512 (adcensus.cu:579) */
#define ADCENSUS_MAX_MEDIAN 11     /* median2d: float xs[11*11] (adcensus.cu:1582) */

typedef void *adcensus_stream_t;   /* cudaStream_t */

/* "libadcensus_b200 <version>"; replaces adcensus.version (adcensus.cu:2055-2059) */
const char *adcensus_version(void);

/* the SM count every launch sized by the SM count uses on the current device: the device's own, or the value of the
 * environment variable ADCENSUS_NUM_SMS (a decimal integer in 1..1024, read once) that tests set to run those launches at
 * other grid sizes.  No output depends on it (DESIGN.md §4). */
int adcensus_num_sms(void);

/* ---- operators of the hot path (one per Lua function) ------------------- */

/* adcensus.StereoJoin(input_L, input_R, output_L, output_R)  adcensus.cu:1455-1498
 * outL[d,y,x] = outR[d,y,x-d] = -sum_c L[c,y,x]*R[c,y,x-d] for x-d >= 0 (fp32 FMA
 * chain, c ascending); other entries are left untouched (caller pre-fills NaN,
 * main.lua:946). */
int adcensus_StereoJoin(const float *input_L, const float *input_R, float *output_L, float *output_R,
			int C, int D, int H, int W, adcensus_stream_t stream);

/* StereoJoin into PITCHED volumes (D, H, ld), ld % 4 == 0, 16-byte aligned outputs, W even, 8-byte aligned features (else
 * ADCENSUS_EINVAL), with the kernels the fused pipeline runs.  Same values as adcensus_StereoJoin bit for bit;
 * additionally output_L[d,y,x] = NaN for x < d (the fill of main.lua:946 for the left volume); output_R's entries with
 * x >= W - d and the padding columns x >= W of both volumes are left untouched. */
int mccnn_stereo_join_pitched(const float *input_L, const float *input_R, float *output_L, float *output_R,
			      int C, int D, int H, int W, int ld, adcensus_stream_t stream);

/* adcensus.cross(x0, out, L1, tau1)  adcensus.cu:280-341; out is (4,H,W) */
int adcensus_cross(const float *x0, float *out, int H, int W, int L1, float tau1, adcensus_stream_t stream);

/* adcensus.cbca(x0c, x1c, vol_in, vol_out, direction)  adcensus.cu:343-400
 * vol_in must not alias vol_out.  Fully asynchronous: the longest arm, which sizes the shared-memory tile, stays on
 * the device -- every candidate kernel is launched with a gate on it and the ones out of range return immediately.
 * Precondition shared with the reference's (compiled-out) assert at adcensus.cu:366: vol_in is finite wherever a support can
 * reach, i.e. on x >= d (direction -1) / x < W - d (direction 1) -- for a fix_border'ed volume that means D <= W - border - 1.
 * Under it the result is bit-identical; a NaN inside the valid part spreads to the outputs of the tile rows that walk over it,
 * not only to the supports that contain it. */
int adcensus_cbca(const float *x0c, const float *x1c, const float *vol_in, float *vol_out,
		  int D, int H, int W, int direction, adcensus_stream_t stream);

/* Same with the kernel chosen on the host: the caller states the longest arm cross() can have produced for these arms,
 * max(L1, 2) (main.lua knows opt.L1).  Arms longer than max_arm (<= 14) are CUT at max_arm (a truncated support, never an
 * out-of-bounds read); state the true bound or use adcensus_cbca.  Asynchronous on `stream`. */
int adcensus_cbca_ex(const float *x0c, const float *x1c, const float *vol_in, float *vol_out,
		     int D, int H, int W, int direction, int max_arm, adcensus_stream_t stream);

/* The two halves of adcensus_cbca for callers that aggregate several times with the same arms
 * (main.lua runs cbca_i1 + cbca_i2 iterations per direction): pack both arm tensors once into
 * `packed` (mccnn_packed_arms_bytes(H, W) bytes of device memory), then iterate.  x0c/x1c are still
 * passed to the aggregation for the generic kernel that serves arms longer than 14 pixels. */
size_t mccnn_packed_arms_bytes(int H, int W);
int mccnn_pack_arms(const float *x0c, const float *x1c, void *packed, int H, int W, adcensus_stream_t stream);
int mccnn_cbca_packed(const void *packed, const float *x0c, const float *x1c, const float *vol_in, float *vol_out,
		      int D, int H, int W, int direction, int max_arm, adcensus_stream_t stream);

/* Constant-work aggregation on PITCHED volumes (csrc/cbca_tma.cu): vol_in / vol_out are (D, H, ld) with a row pitch
 * ld >= W, ld % 4 == 0 and 16-byte aligned bases, so that the plane tiles can be staged by TMA.  NOT bit-exact with
 * the reference: every support row's run is a difference of row prefix sums and the rows are combined through
 * running sums down the column (~45 instructions per output instead of ~200, ~1e-6 relative to the tap-by-tap
 * sums, NaN positions identical); it serves the 1e-4 contract of the north star for float aggregation.  x0c / x1c
 * must be cross() outputs with arms of at most max_arm <= 14 pixels, and the volume must be finite on its valid
 * part (D <= W - border - 1 for a fix_border'ed volume).  The padding columns of vol_out are left untouched. */
int mccnn_cbca_fast_pitched(const float *x0c, const float *x1c, const float *vol_in, float *vol_out,
			    int D, int H, int W, int ld, int direction, int max_arm, adcensus_stream_t stream);

/* The two halves of mccnn_cbca_fast_pitched: pack both arm tensors once (mccnn_packed_hv_bytes(H, W) bytes), then iterate. */
size_t mccnn_packed_hv_bytes(int H, int W);
int mccnn_pack_arms_hv(const float *x0c, const float *x1c, void *hv, int H, int W, adcensus_stream_t stream);
int mccnn_cbca_fast_pitched_packed(const void *hv, const float *vol_in, float *vol_out,
				   int D, int H, int W, int ld, int direction, int max_arm, adcensus_stream_t stream);

/* adcensus.sgm2(x0, x1, input, output, tmp, pi1, pi2, tau_so, alpha1, sgm_q1,
 *               sgm_q2, direction)  adcensus.cu:535-697
 * input/output are (H,W,D); output is accumulated into (+=) in the order right,
 * left, down, up.  tmp (>= W*D floats) is the reference's line-state scratch; it
 * is accepted for signature parity and may be NULL (state lives on chip). */
int adcensus_sgm2(const float *x0, const float *x1, const float *input, float *output, float *tmp,
		  int H, int W, int D, float pi1, float pi2, float tau_so, float alpha1,
		  float sgm_q1, float sgm_q2, int direction, adcensus_stream_t stream);

/* Band-wise sgm2 for the row-band / column-band multi-GPU split: x0, x1 are the FULL Ht x Wt images,
 * input/output this GPU's band volume (H,W,D) at image offset (yoff, xoff); pass_mask selects scan
 * directions (bit 0 right, 1 left, 2 down, 3 up; run in that order).  A band must hold whole scanlines
 * of every selected pass (row bands for bits 0-1, column bands for bits 2-3).  zero_out != 0: `output`
 * is known to be zero on entry. */
int mccnn_sgm2_band(const float *x0, const float *x1, const float *input, float *output,
		    int H, int W, int D, int Ht, int Wt, int yoff, int xoff,
		    float pi1, float pi2, float tau_so, float alpha1, float sgm_q1, float sgm_q2,
		    int direction, int pass_mask, int zero_out, adcensus_stream_t stream);

/* The fused pipeline's sgm2: all four directions of the whole image into `output` as if it were zero on entry (it is
 * written, never read), bit-identical to mccnn_sgm2_band with pass_mask 15 and zero_out.  Forward scans store their line
 * states in `scratch` (16-byte aligned) and the backward scans recompute from them, 7 volume passes instead of 11.
 * mccnn_sgm2_ckpt_bytes gives the scratch it needs (0: not at this shape); with less, it runs the 11-pass kernels. */
size_t mccnn_sgm2_ckpt_bytes(int H, int W, int D);
int mccnn_sgm2_ckpt(const float *x0, const float *x1, const float *input, float *output, void *scratch,
		    size_t scratch_bytes, int H, int W, int D, float pi1, float pi2, float tau_so, float alpha1,
		    float sgm_q1, float sgm_q2, int direction, adcensus_stream_t stream);

/* Wavefront split of sgm2 over ROW bands (the multi-GPU single-volume path, rowband.py).  Build the penalty-class tables
 * of the image pair once (mccnn_sgm_tables_bytes bytes; classes + the selector words of one `direction`), then run the
 * passes band by band on (H,W,D) band volumes at image row offset yoff: horizontal passes (bits 0-1) are band-local; a
 * vertical pass (bit 2 down or bit 3 up, ONE per call when chained) over the columns [xa, xb) takes the line state of the
 * row before the band from state_in (NULL only where the scan starts at the image border) and leaves the state of the
 * band's last row in state_out: [W][mccnn_sgm_state_pitch(D)] floats.  Same arithmetic and accumulation order as
 * adcensus_sgm2: chained over all bands the result is bit-identical to the whole-image call. */
size_t mccnn_sgm_tables_bytes(int Ht, int Wt, int D);
int mccnn_sgm_state_pitch(int D);
int mccnn_sgm_tables_build(const float *x0, const float *x1, void *tab, int Ht, int Wt, int D, float tau_so,
			   int direction, adcensus_stream_t stream);
int mccnn_sgm2_rows(const void *tab, const float *input, float *output, int H, int W, int D, int Ht, int yoff,
		    float pi1, float pi2, float tau_so, float alpha1, float sgm_q1, float sgm_q2,
		    int direction, int pass_mask, int zero_out, int xa, int xb,
		    const float *state_in, float *state_out, adcensus_stream_t stream);

/* adcensus.outlier_detection(d0, d1, outlier, disp_max)  adcensus.cu:878-918 */
int adcensus_outlier_detection(const float *d0, const float *d1, float *outlier,
			       int H, int W, int disp_max, adcensus_stream_t stream);

/* adcensus.interpolate_occlusion(d0, outlier) -> out  adcensus.cu:1079-1125
 * (the Lua face allocates `out` like new_tensor_like, adcensus.cu:40-45) */
int adcensus_interpolate_occlusion(const float *d0, const float *outlier, float *out,
				   int H, int W, adcensus_stream_t stream);

/* adcensus.interpolate_mismatch(d0, outlier) -> out  adcensus.cu:1001-1077 */
int adcensus_interpolate_mismatch(const float *d0, const float *outlier, float *out,
				  int H, int W, adcensus_stream_t stream);

/* adcensus.subpixel_enchancement(d0, c2, disp_max) -> out  adcensus.cu:1205-1239
 * c2 is the (disp_max,H,W) cost volume */
int adcensus_subpixel_enchancement(const float *d0, const float *c2, float *out,
				   int H, int W, int disp_max, adcensus_stream_t stream);

/* adcensus.median2d(img, kernel_size) -> out  adcensus.cu:1575-1613; odd ksize <= 11 */
int adcensus_median2d(const float *img, float *out, int H, int W, int kernel_size, adcensus_stream_t stream);

/* adcensus.mean2d(img, kernel, alpha2) -> out  adcensus.cu:1241-1282
 * kernel is (ksize,ksize), ksize odd */
int adcensus_mean2d(const float *img, const float *kernel, float *out, int H, int W, int ksize,
		    float alpha2, adcensus_stream_t stream);

/* adcensus.Normalize_forward(input, norm, output)  adcensus.cu:1284-1333
 * input/output (N,C,H,W), norm (N,1,H,W) */
int adcensus_Normalize_forward(const float *input, float *norm, float *output,
			       int N, int C, int H, int W, adcensus_stream_t stream);

/* adcensus.spatial_argmin(input, output)  adcensus.cu:244-278
 * input (N,D,H,W) -> output (N,1,H,W), 1-based, strict <, NaN skipped */
int adcensus_spatial_argmin(const float *input, float *output, int N, int D, int HW, adcensus_stream_t stream);

/* adcensus.ad / adcensus.census  adcensus.cu:62-175 (net-free cost volumes; x0,x1 (nch,H,W)) */
int adcensus_ad(const float *x0, const float *x1, float *out, int D, int H, int W, int direction,
		adcensus_stream_t stream);
int adcensus_census(const float *x0, const float *x1, float *out, int D, int nch, int H, int W,
		    int direction, adcensus_stream_t stream);

/* ---- the Lua-side tensor ops of stereo_predict (cutorch in the reference) - */

/* vols:fill(0/0)  main.lua:946 */
int mccnn_fill_nan(float *p, size_t n, adcensus_stream_t stream);
/* the part of that fill StereoJoin does not overwrite: NaN where x < d (left volume) and x >= W - d
 * (right volume); what the fused pipeline uses instead of filling 2V bytes */
int mccnn_fill_invalid(float *volL, float *volR, int D, int H, int W, adcensus_stream_t stream);
/* fix_border(net, vol, direction)  main.lua:922-927; n = (window-1)/2 */
int mccnn_fix_border(float *vol, int D, int H, int W, int n, int direction, adcensus_stream_t stream);
/* vol:transpose(2,3):transpose(3,4):clone()  main.lua:1008   (D,H,W) -> (H,W,D) */
int mccnn_transpose_dhw_to_hwd(const float *in, float *out, int D, int H, int W, adcensus_stream_t stream);
/* vol:copy(out:transpose(3,4):transpose(2,3)):div(4)  main.lua:1020   (H,W,D) -> (D,H,W), /4 */
int mccnn_transpose_hwd_to_dhw_div4(const float *in, float *out, int D, int H, int W, adcensus_stream_t stream);
/* _, d = torch.min(vol, 2); d:add(-1)  main.lua:1049-1050: 0-based argmin as float,
 * first minimum, NaN skipped (the in-repo statement is spatial_argmin) */
int mccnn_argmin(const float *vol, float *disp, int D, int HW, adcensus_stream_t stream);
/* the same three ops on the fused pipeline's pitched (D, H, ld) volumes: (D,H,ld) -> (H,W,D); (H,W,D) -> (D,H,ld) with /4;
 * first minimum over D */
int mccnn_transpose_dhw_pitched_to_hwd(const float *in, float *out, int D, int H, int W, int ld, adcensus_stream_t stream);
int mccnn_transpose_hwd_to_dhw_pitched_div4(const float *in, float *out, int D, int H, int W, int ld, adcensus_stream_t stream);
int mccnn_argmin_pitched(const float *vol, float *disp, int D, int H, int W, int ld, adcensus_stream_t stream);
/* gaussian(sigma)  main.lua:528-540: HOST helper; returns ksize, fills out (ksize*ksize) if non-NULL */
int mccnn_gaussian(double sigma, float *out_host);

/* ---- fused stereo_predict (main.lua:929-1082, arch 'fast') ---------------- */

typedef struct mccnn_params {
	int L1;
	float tau1;
	int cbca_i1, cbca_i2;
	float pi1, pi2, sgm_q1, sgm_q2, alpha1, tau_so;
	int sgm_i;
	double blur_sigma;
	float blur_t;
	int border;    /* fix_border n (4 for the 4-layer 3x3 tower, main.lua:382-391,923) */
	int lr_check;  /* 1: kitti / kitti2015 (main.lua:1054); 0: mb */
	/* main.lua's -sm_terminate / -sm_skip (main.lua:953-1082): an MCCNN_SM_* code each, 0 = the full chain.  A step
	 * runs while no earlier -sm_terminate step has been passed and it is not the skipped one; terminate occlusion /
	 * mismatch and skip occlusion act only with the LR check.  When the chain stops early, disp receives the map
	 * main.lua returns (the 0-based argmin of the left volume for terminate cnn / cbca1 / sgm / cbca2). */
	int sm_terminate;  /* MCCNN_SM_CNN .. MCCNN_SM_MEDIAN */
	int sm_skip;       /* MCCNN_SM_CBCA, _SGM, _OCCLUSION, _SUBPIXEL, _MEDIAN, _BILATERAL */
} mccnn_params;

/* Stage codes of mccnn_params.sm_terminate / sm_skip, named after main.lua's option values.  Terminate accepts cnn, cbca1,
 * sgm, cbca2, occlusion, mismatch, subpixel_enchancement and median; skip accepts cbca, sgm, occlusion,
 * subpixel_enchancement, median and bilateral.  Any other code is refused (ADCENSUS_EINVAL). */
enum {
	MCCNN_SM_NONE = 0,
	MCCNN_SM_CNN = 1,        /* terminate: the argmin of the raw volume */
	MCCNN_SM_CBCA1 = 2,      /* terminate: after cross + the first CBCA block */
	MCCNN_SM_SGM = 3,        /* terminate / skip: SGM */
	MCCNN_SM_CBCA2 = 4,      /* terminate: after the second CBCA block */
	MCCNN_SM_OCCLUSION = 5,  /* terminate / skip (both interpolations): LR check only */
	MCCNN_SM_MISMATCH = 6,   /* terminate: LR check only */
	MCCNN_SM_SUBPIXEL = 7,   /* terminate / skip: subpixel_enchancement */
	MCCNN_SM_MEDIAN = 8,     /* terminate / skip: median2d */
	MCCNN_SM_BILATERAL = 9,  /* skip: mean2d */
	MCCNN_SM_CBCA = 10       /* skip: the cross arms and both CBCA blocks */
};

typedef struct mccnn_pipeline mccnn_pipeline;

/* Allocates every device buffer the pipeline needs for (C,D,H,W) on `device`. */
int mccnn_pipeline_create(mccnn_pipeline **out, int C, int D, int H, int W,
			  const mccnn_params *params, int device);
void mccnn_pipeline_destroy(mccnn_pipeline *p);
size_t mccnn_pipeline_device_bytes(const mccnn_pipeline *p);
/* CBCA mode of the pipeline's iterations: 1 (default) = constant-work aggregation (mccnn_cbca_fast_pitched: volumes within
 * the north star's 1e-4 of the reference, measured ~1e-6; disparity map identical except at isolated near-ties) for presets
 * whose arms are at most 5 pixels long, the exact kernels for longer arms; 0 = exact, every output bit-identical to the
 * reference.  ADCENSUS_CBCA_EXACT=1 in the environment makes 0 the default. */
void mccnn_pipeline_set_cbca_mode(mccnn_pipeline *p, int mode);
int mccnn_pipeline_get_cbca_mode(const mccnn_pipeline *p);
/* Schedule of the two directions of main.lua:955.  1 or 2 (the default, set at create time when the extra buffers fit):
 * concurrent -- direction -1 on a side stream with its own 2V + tables, started when direction +1 reaches its SGM phase,
 * and the permute / SGM phases on high-priority streams.  0: sequential on one stream, 4V of volume buffers instead of 6V.
 * Results are identical in every mode (same kernels, same data); only the schedule and the memory footprint change.
 * Returns 0 or an error. */
int mccnn_pipeline_set_overlap(mccnn_pipeline *p, int mode);
/* number of kernel launches the last run issued (for bench.py's gpu_launches); fewer when sm_terminate / sm_skip drop steps */
int mccnn_pipeline_launches_per_run(const mccnn_pipeline *p);
/* Re-targets a created pipeline to another parameter set without allocating its volumes again (a parameter search runs
 * many sets over the same images).  Checked like mccnn_pipeline_create (ADCENSUS_EINVAL; border + 1 must not exceed the
 * created W).  HOST-SYNCHRONOUS: waits for all work enqueued on the pipeline's device before anything an enqueued run reads
 * changes.  The Gaussian buffer grows only when blur_sigma needs a larger kernel (sigma 10 -> 61 x 61).  Applies to every
 * twin lane of the batch entry points that exists; lanes created later inherit the new parameters.  Every later run gives
 * the same bits as a pipeline created with these parameters, in the same CBCA mode and overlap mode.  On an
 * error (a CUDA error, or no memory for a larger Gaussian) the pipeline must be re-targeted again or destroyed. */
int mccnn_pipeline_set_params(mccnn_pipeline *p, const mccnn_params *params);

/* Device-resident inputs: featL/featR (C,H,W) unit-norm tower outputs, imgL/imgR
 * (H,W) standardised images.  disp (H,W) device; volL/volR (D,H,W) device or NULL
 * (what `-a predict` writes to left.bin/right.bin).  Asynchronous on `stream`. */
int mccnn_pipeline_run(mccnn_pipeline *p, const float *featL, const float *featR,
		       const float *imgL, const float *imgR, float *disp,
		       float *volL, float *volR, adcensus_stream_t stream);

/* Run at (H, W, D) with H <= the created H, W <= the created W, D <= the created D; C and params as created, so that
 * one pipeline created at the largest shape of a dataset serves every image of it (KITTI widths, Middlebury sizes and
 * disparity ranges) without allocating.  featL/featR (C,H,W), imgL/imgR (H,W), disp (H,W), volL/volR (D,H,W) or NULL,
 * all contiguous at the RUN shape.  Same results, bit for bit, as mccnn_pipeline_run on a pipeline created at (C, D, H, W)
 * with the same params, CBCA mode and overlap mode.  ADCENSUS_ELIMIT if the shape exceeds the created one,
 * ADCENSUS_EINVAL for H, W or D < 1 or border + 1 > W; nothing is launched then.  Asynchronous on `stream`.
 * The batch, host and twin-lane entry points (mccnn_pipeline_run_batch / _run_host / _run_host_batch) always run at the
 * created shape. */
int mccnn_pipeline_run_shape(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR,
			     const float *imgL, const float *imgR, float *disp, float *volL, float *volR,
			     adcensus_stream_t stream);

/* The chain of mccnn_pipeline_run_shape from given cost volumes on: volL / volR (D,H,W) contiguous at the run shape, what
 * main.lua holds at :986 -- NaN where the reference leaves its fill, fix_border (:948-949 / :981) already applied by the
 * caller (the fast net's StereoJoin volumes, the scorer head's, or adcensus_ad / adcensus_census outputs).  They are copied
 * into the private pitched buffers (not modified), then cross / CBCA / SGM / ... run exactly as in mccnn_pipeline_run_shape,
 * same bits for the same volumes.  volR may be NULL when lr_check == 0 and outR == NULL (Middlebury: only direction -1 is
 * consumed, main.lua:954-955).  imgL/imgR/disp (H,W); outL/outR (D,H,W) or NULL.  Shape limits and error codes as
 * mccnn_pipeline_run_shape; ADCENSUS_EINVAL also for a NULL volR that is needed.  Asynchronous on `stream`. */
int mccnn_pipeline_run_volumes(mccnn_pipeline *p, int H, int W, int D, const float *volL, const float *volR,
			       const float *imgL, const float *imgR, float *disp, float *outL, float *outR,
			       adcensus_stream_t stream);

/* ---- confidence, LR map, sparse maps and sparsification counts (csrc/confidence.cu; DESIGN §19) ---------------------------
 * An addition beyond the reference.  Margin confidence of a (D,H,W) volume at each pixel: d1 = the arg-min of
 * mccnn_argmin_pitched (first strict minimum, NaN skipped, 0 when nothing is below +inf) with value c1; c2 = the minimum by
 * the same rule over the d with |d - d1| >= 2; conf = c2 - c1 in float when both are below +inf, else 0.  The confidence
 * belongs to the integer winner: sub-pixel refinement, median and bilateral filtering move the disparity, not its confidence.
 *
 * mccnn_pipeline_run_shape_conf / _run_volumes_conf: mccnn_pipeline_run_shape / _run_volumes that also write conf (H,W),
 * the margin confidence of the final left volume (what volL / outL receives), and lr (H,W), main.lua:1056's outlier map
 * (0 consistent, 1 mismatch, 2 occlusion) of the two winner-take-all maps; for lr, direction +1 and the LR check run even
 * when -sm_terminate / -sm_skip would skip them.  conf and lr may be NULL; with both NULL the calls are the plain ones (same
 * launches, same bits), and disp never changes with them.  ADCENSUS_EINVAL, before any launch, for lr with lr_check == 0
 * and as the plain calls. */
int mccnn_pipeline_run_shape_conf(mccnn_pipeline *p, int H, int W, int D, const float *featL, const float *featR,
				  const float *imgL, const float *imgR, float *disp, float *conf, float *lr, float *volL,
				  float *volR, adcensus_stream_t stream);
int mccnn_pipeline_run_volumes_conf(mccnn_pipeline *p, int H, int W, int D, const float *volL, const float *volR,
				    const float *imgL, const float *imgR, float *disp, float *conf, float *lr, float *outL,
				    float *outR, adcensus_stream_t stream);
/* The arg-min (disp) and the margin confidence (conf) of a contiguous (D,H,W) volume in one read; disp bit-identical to
 * mccnn_argmin.  H <= 65535. */
int mccnn_margin_confidence(const float *vol, float *disp, float *conf, int D, int H, int W, adcensus_stream_t stream);
/* out = disp at the n_keep pixels of largest conf (ties: lower row-major index first), `invalid` elsewhere.  Pixels are
 * ordered by conf's float bits, which order like the values (NaN above +inf).  1 <= n_keep <= H*W (else ADCENSUS_EINVAL),
 * H*W < 2^32 (else ADCENSUS_ELIMIT); out must not alias disp or conf.  Exact and deterministic.  Asynchronous. */
int mccnn_sparsify(const float *disp, const float *conf, float *out, int H, int W, long long n_keep, float invalid,
		   adcensus_stream_t stream);
/* The counts of the sparsification curve of pred against gt (H,W): counts[0] = M, the pixels with gt != 0 (main.lua:1230);
 * counts[1] = B, the bad ones among them (|gt - pred| > err_at); counts[1 + k], k = 1..20 = the bad ones among the first
 * n_k = ceil(k M / 20) of the M pixels ordered as mccnn_sparsify orders them.  counts: 22 long longs in device memory.
 * Exact and deterministic.  Asynchronous. */
int mccnn_sparsification_counts(const float *pred, const float *conf, const float *gt, int H, int W, float err_at,
				long long *counts, adcensus_stream_t stream);

/* Host-buffer call (what a non-CUDA caller binds): copies inputs H2D, runs,
 * copies disp back, and returns after the result is in disp_host. */
int mccnn_pipeline_run_host(mccnn_pipeline *p, const float *featL_host, const float *featR_host,
			    const float *imgL_host, const float *imgR_host, float *disp_host);

/* Same for n pairs (arrays of n host pointers each): the H2D copy of pair i+1 and the D2H copy of
 * pair i-1 overlap the kernels of pair i (two staging slots, a copy stream and a compute stream).
 * Host buffers should be pinned for the overlap to materialise.  Returns when all n results are
 * in their host buffers. */
int mccnn_pipeline_run_host_batch(mccnn_pipeline *p, int n, const float *const *featL_host,
				  const float *const *featR_host, const float *const *imgL_host,
				  const float *const *imgR_host, float *const *disp_host);

/* Operator-level calls take their scratch (SGM tables, packed arms) stream-ordered from the device's default memory pool; the
 * library raises that pool's release threshold to 2 GiB (never lowers it) so that repeated calls reuse the memory.
 * adcensus_trim_scratch() hands everything unused back to the driver. */
int adcensus_trim_scratch(void);

/* n device-resident pairs (arrays of n device pointers each), ordered on `stream` as a whole.  Pairs alternate between two
 * lanes (two buffer sets on internal streams, created on first use; one lane if the second does not fit), so that one
 * pair's low-occupancy post-processing tail overlaps the next pair's volume kernels.  Results identical to n calls of
 * mccnn_pipeline_run. */
int mccnn_pipeline_run_batch(mccnn_pipeline *p, int n, const float *const *featL, const float *const *featR,
			     const float *const *imgL, const float *const *imgR, float *const *disp, adcensus_stream_t stream);

/* ---- the accurate ('slow') architecture's scorer head (csrc/scorer_head.cu) -------------------------------------
 * Replaces the per-disparity loop of main.lua:958-984 over net_te2 (main.lua:688-695: l2 x [SpatialConvolution1_fw,
 * ReLU], SpatialConvolution1_fw(nh2 -> 1), Sigmoid; SpatialConvolution1_fw.lua:11-31 = addmm + bias per pixel) by one
 * fused wgmma kernel.  Outside libadcensus.so in the reference (a Lua nn module chain), hence a mccnn_* entry.
 * W[i] (out_i x in_i, row-major) and b[i] (out_i), i = 0 .. l2, DEVICE pointers in net_te2's order: layer 0 is
 * (nh2 x 2 fm), layers 1 .. l2-1 (nh2 x nh2), layer l2 (1 x nh2).  Limits: l2 <= 4, nh2 a multiple of 128 and <= 384,
 * fm a multiple of 8 with 2 fm <= 384 (the kitti / kitti2015 / mb nets: fm 112, nh2 384, l2 3..4). */
typedef struct mccnn_scorer_head mccnn_scorer_head;
int mccnn_scorer_head_create(mccnn_scorer_head **out, int fm, int nh2, int l2, const float *const *W, const float *const *b,
			     int device, adcensus_stream_t stream);
void mccnn_scorer_head_destroy(mccnn_scorer_head *h);
/* featL / featR: (fm, H, W) tower outputs; volL / volR: (D, H, W), either may be NULL.  Writes volL[d, y, x] for x >= d and
 * volR[d, y, x - d] (the same score, main.lua:976); all other entries keep the caller's NaN fill (:962); fix_border (:981)
 * is the caller's next call.  nterms 3: bf16-split operands, fp32-grade (1e-4 contract); 1: plain bf16. */
int mccnn_scorer_head_forward(const mccnn_scorer_head *h, const float *featL, const float *featR, float *volL, float *volR,
			      int H, int W, int D, int nterms, adcensus_stream_t stream);

/* ---- the feature tower in-library (csrc/feature_tower.cu) --------------------------------------------
 * net_te at test time (main.lua:682-686 arch 'slow', 726-749 arch 'fast'): l1 x cudnn.SpatialConvolution(3x3, stride 1,
 * pad 1) with ReLU between the layers; arch 'fast' ends with Normalize2 (adcensus.cu:1284-1308) instead of a ReLU.
 * W[i] (fm, cin_i, 3, 3) row-major and b[i] (fm), i = 0 .. l1-1, DEVICE pointers (cudnn.SpatialConvolution's weight / bias).
 * Layer 1 (n_in = 1 or 3 planes) is exact fp32; the fm -> fm layers are wgmma implicit GEMMs (nterms 3: bf16-split
 * operands, fp32-grade; 1: plain bf16).  Limits: fm a multiple of 16 and <= 128, l1 <= 8. */
typedef struct mccnn_feature_tower mccnn_feature_tower;
int mccnn_feature_tower_create(mccnn_feature_tower **out, int n_in, int fm, int l1, int relu_last, int normalize,
			       const float *const *W, const float *const *b, int device, adcensus_stream_t stream);
void mccnn_feature_tower_destroy(mccnn_feature_tower *h);
/* img (nimg, n_in, H, W) -> out (nimg, fm, H, W); nimg = 2 for x_batch of main.lua:944. */
int mccnn_feature_tower_forward(const mccnn_feature_tower *h, const float *img, float *out, int nimg, int H, int W,
				int nterms, adcensus_stream_t stream);

/* ---- KITTI label cleaning and training-sample lists (csrc/preprocess.cu, preprocess_kitti.lua:95-116) ----------------
 * Stacks are (N, 1, H, W) disparity maps, treated as N*H rows of W columns as the reference does (x = index % W); the three
 * cleaning operators work in place.  Not registered in the Lua face yet (csrc/lua_face.cu still names them
 * "not implemented"). */

/* adcensus.remove_nonvisible(y)  adcensus.cu:1723-1745: y[.., x] >= x -> 0 */
int adcensus_remove_nonvisible(float *y, int N, int H, int W, adcensus_stream_t stream);

/* adcensus.remove_occluded(y)  adcensus.cu:1747-1771: y[.., x] -> 0 if some i >= 1, x + i < W, has i - y[x+i] < -y[x].
 * Computed as one reverse suffix minimum of j - y[j] per row (DESIGN.md).  PRECONDITION for bit-identity with the reference:
 * every y is >= 0 and every x - y[x] is exact in fp32 -- true for any map readPNG16 produces (multiples of 1/256 in [0, 256))
 * with W <= 2^15.  ADCENSUS_ELIMIT for W > 32768. */
int adcensus_remove_occluded(float *y, int N, int H, int W, adcensus_stream_t stream);

/* adcensus.remove_white(x, y)  adcensus.cu:1773-1796: y -> 0 where x == 255 (x has y's N*H*W elements) */
int adcensus_remove_white(const float *x, float *y, int N, int H, int W, adcensus_stream_t stream);

/* The sample lists nnz_tr / nnz_te of preprocess_kitti.lua:95-116 in two calls.  disp (n, 1, H, W) training maps (not
 * modified: the cleaning runs on an on-chip copy), x0 (at least n, 1, H, W) their standardised left images, is_te (n) int32
 * flags (1: image i is in the validation split te).  Per map: remove_nonvisible, remove_occluded, remove_white(x0[i]); then
 * every entry d > 0.5 becomes the float row (i + 1, y, x, d) of nnz_te if is_te[i] else nnz_tr, ordered by image, then row,
 * then column -- make_dataset2's order (adcensus.cu:1900-1929).  Same precondition as adcensus_remove_occluded;
 * ADCENSUS_ELIMIT for W > 32768 or n*H*W >= 2^31.
 *   mccnn_kitti_nnz_count writes the two row counts to counts[0] (nnz_tr) and counts[1] (nnz_te), DEVICE int64;
 *   mccnn_kitti_nnz_fill writes the rows ((rows, 4) float32, 16-byte aligned); rows past cap_tr / cap_te are dropped, and a
 *   buffer may be NULL when its cap is 0.  Size the buffers with the count call. */
int mccnn_kitti_nnz_count(const float *disp, const float *x0, const int *is_te, int n, int H, int W, long long *counts,
			  adcensus_stream_t stream);
int mccnn_kitti_nnz_fill(const float *disp, const float *x0, const int *is_te, int n, int H, int W, float *nnz_tr,
			 long long cap_tr, float *nnz_te, long long cap_te, adcensus_stream_t stream);

/* ---- the image front end of main.lua -a predict and predict_kitti.lua's error (csrc/frontend.cu) ------------------------
 * All pointers are DEVICE pointers. */

/* frontend.make_batch (main.lua:1085-1100) on one pair: left / right the decoded 8-bit views, (H, W) grey (nch 1) or (H, W, 3)
 * interleaved R, G, B (nch 3, through image.rgb2y); x_batch (2, 1, H, W) float32, bit-identical to frontend.make_batch.
 * Y = 0.299 R, + 0.587 G, + 0.114 B, each product and sum rounded in fp32.  Per view, frontend.standardise: m = sum(y) / n,
 * y' = y + f32(-m) in fp32, m2 = sum(y') / n, var = sum((y' - m2)^2) / (n - 1), out = y' / f32(sqrt(var)), every sum
 * numpy's pairwise float64 sum over the view in memory order.  stats (2, 3) float64 receives (m, m2, var) per view: a
 * constant view has var == 0 (its x_batch plane is then not finite) and the caller must refuse it, as standardise does.
 * H * W >= 2 (else ADCENSUS_EINVAL), H * W * nch < 2^31 (else ADCENSUS_ELIMIT). */
int mccnn_frontend_batch(const unsigned char *left, const unsigned char *right, int nch, int H, int W, float *x_batch,
			 double *stats, adcensus_stream_t stream);

/* dataio.bad_pixel_rate's counts for one map (predict_kitti.lua:62-70): disp (H, W) float32, gt (H, W) the PNG16 ground
 * truth as stored (uint16, disparity * 256, 0 = invalid).  counts[0] = #(gt != 0 and |gt / 256 - disp| > err_at) in fp32
 * (a NaN disparity is not bad), counts[1] = #(gt != 0); DEVICE int64, overwritten.  The error is counts[0] / counts[1]. */
int mccnn_kitti_error_count(const float *disp, const unsigned short *gt, int H, int W, float err_at, long long *counts,
			    adcensus_stream_t stream);

/* ---- Middlebury views, halving, masks and training-sample lists (csrc/preprocess_mb.cu, preprocess_mb.py) ---------------
 * All pointers are DEVICE pointers; images are 8-bit (n, H, W, 3) in R, G, B order (a grey file replicated to three
 * channels, as cv2.imread does). */

/* read_im (preprocess_mb.py:85-97) on n views: out (n, nchannel, H, W) float32.  nchannel 1: cv2's BGR2GRAY,
 * fma(R, .299, fma(B, .114, G * .587)) in fp32; 3: the R, G, B planes.  Then (x - mean) / std exactly as numpy's float32
 * x.mean() and x.std() (pairwise sums in memory order, pixels with interleaved channels): bit-identical.  n <= 65535,
 * H * W * 3 < 2^31 (else ADCENSUS_ELIMIT). */
int mccnn_mb_views(const unsigned char *rgb, float *out, int n, int H, int W, int nchannel, adcensus_stream_t stream);

/* `convert X -resize 50%` restated, NOT bit-pinned against ImageMagick: (n, H, W, 3) -> (n, H/2, W/2, 3).  Lanczos-3
 * L(t) = sinc(t) sinc(t/3); output x reads source 2x-5 .. 2x+6 with weights L((j + 0.5 - (2x + 1)) / 2), taps outside the
 * image dropped and the rest renormalised; rows first, then columns, in fp32; rounded half up, clamped to [0, 255].  H and
 * W must be even (ADCENSUS_EINVAL otherwise). */
int mccnn_mb_half_image(const unsigned char *in, unsigned char *out, int n, int H, int W, adcensus_stream_t stream);

/* load_pfm(.., True) (preprocess_mb.py:13-26) on n top-down maps: out (n, H/2, W/2) = the second smallest of each 2x2 block
 * of in / 2 in np.sort's order (-inf < finite < inf < NaN).  H and W must be even. */
int mccnn_mb_half_disp(const float *in, float *out, int n, int H, int W, adcensus_stream_t stream);

/* `computemask d0 [d0y] d1 -1` restated, NOT pinned against the MiddEval3 SDK: mask (H, W) bytes = 0 where d0 is not
 * finite; else x1 = floor(x - d0 + 0.5), y1 = floor(y + d0y + 0.5) (d0y may be NULL: 0), in fp64; 128 when (x1, y1) is
 * outside the frame (or d0y not finite) or when not |d0 - d1[y1, x1]| <= 1 (inf and NaN on the right fail); else 255. */
int mccnn_mb_mask(const float *d0, const float *d0y, const float *d1, int H, int W, unsigned char *mask,
		  adcensus_stream_t stream);

/* The training rows of one map (preprocess_mb.py:177-182) in two calls:
 *   mccnn_mb_nnz_count writes the number of mask == 255 pixels to *count (DEVICE int64);
 *   mccnn_mb_nnz_fill writes dispnoc (H, W) = d0 where mask == 255, else 0, and the float rows (image, y, x, d0) of those
 *   pixels in row-major order to nnz ((rows, 4) float32, 16-byte aligned); rows past cap are dropped, nnz may be NULL when
 *   cap is 0.  image is 1-based, <= 2^24. */
int mccnn_mb_nnz_count(const unsigned char *mask, int H, int W, long long *count, adcensus_stream_t stream);
int mccnn_mb_nnz_fill(const float *d0, const unsigned char *mask, int H, int W, int image, float *dispnoc, float *nnz,
		      long long cap, adcensus_stream_t stream);

/* ---- training of the fast architecture (csrc/train.cu, train.py; main.lua:602-890) ------------------------------------
 * Patches are ws x ws, ws = 1 + 2 l1; a batch of bs pairs is N = 2 bs patches, sample i owning patches 4i .. 4i + 3
 * (main.lua:843-846).  Pointers may be host or device unless noted (copies use cudaMemcpyDefault). */

/* One patch of make_patch (main.lua:607-619): m the forward 2x3 matrix as stored in the FloatTensor, contrast and
 * brightness as float, image the 0-based index into the trainer's or sampler's pair table, view 0 = the pair's x0, 1 = its
 * x1. */
typedef struct {
	float m[6];
	float contrast, brightness;
	int image, view;
} mccnn_warp;

/* One stereo pair the sampler reads: two DEVICE float32 planes of H x W (row-major, contiguous), 1 <= H, W <= 32767.
 * Pairs of one table may differ in size (Middlebury: one pair per image, light and exposure; main.lua:828-841). */
typedef struct {
	const float *x0, *x1;
	int H, W;
} mccnn_train_pair;

/* What mccnn_trainer_create builds: the arch, main.lua's options of that arch, and the trainer's rank of world ranks. */
typedef struct {
	int slow;             /* 0: arch 'fast', 1: arch 'slow' */
	int l1, fm, bs;
	float mom;
	float margin;         /* 'fast' only (Margin2) */
	int pow;              /* 'fast' only: 1 or 2 */
	int l2, nh2;          /* 'slow' only */
	int chunk, loss_cap;
	int rank, world;      /* world 1 (rank 0): one GPU; >= 2: a data-parallel shard */
} mccnn_trainer_config;

/* The sampler alone: out (n, ws, ws) = warpAffine(X, m, (ws, ws), INTER_CUBIC, BORDER_CONSTANT 0) * contrast +
 * brightness, bit-identical to OpenCV's float path as oracle/train.py restates it, on a DEVICE table of n_pairs pairs: the
 * source X of warps[i] is pairs[image].x0 (view 0) or .x1 (view 1), and its constant-0 border is that pair's own H x W.
 * DEVICE pointers; a pair index outside [0, n_pairs) gives a NaN patch.  The table is read back to the host once to check
 * it (ADCENSUS_EINVAL for a null plane or a size < 1, ADCENSUS_ELIMIT above 32767), so the call waits for `stream`. */
int mccnn_train_sample_pairs(const mccnn_train_pair *pairs, int n_pairs, const mccnn_warp *warps, int n, int ws, float *out,
			     adcensus_stream_t stream);

typedef struct mccnn_trainer mccnn_trainer;

/* The trainer cfg describes, on `device`, sampling from a table of stereo pairs: `pairs` is a HOST array of n_pairs
 * records, copied into trainer-owned device memory; the planes it points to are kept by the caller for the trainer's
 * lifetime.  A warp's image is an index into this table.
 *
 * 'fast' (slow 0): net_tr of l1 valid 3x3 convolutions 1 -> fm -> .. -> fm, ReLU between them, Normalize2, StereoJoin1,
 * with Margin2(margin, pow).
 * 'slow' (slow 1, main.lua:663-677): l1 valid 3x3 convolutions 1 -> fm -> .. -> fm with a ReLU after every one,
 * Reshape(bs, 2 fm) (row r = the features of patches 2r and 2r + 1), l2 x [Linear(in, nh2), ReLU], Linear(nh2, 1), Sigmoid,
 * then BCECriterion2 against the targets 0, 1, 0, 1, ... (main.lua:848-849); the loss of a step is BCECriterion2's output.
 * Both with momentum `mom`, for batches of bs pairs.  Parameters, momenta and gradients are one flat fp32 vector each: per
 * tower layer W (fm, cin, 3, 3) then b (fm), layer 1 first, then ('slow') per Linear W (out, in) followed by b (out), in
 * main.lua's order; all start at 0.  fp32 on the CUDA cores with fixed reduction orders and no floating-point atomics, so
 * equal inputs give equal bits.  `chunk` bounds the steps of one mccnn_trainer_run or mccnn_trainer_shard_begin,
 * `loss_cap` the per-step losses kept between two mccnn_trainer_reset_losses.
 *
 * The arguments are checked before the first CUDA call, and *h is NULL after any failure.  ADCENSUS_EINVAL: a null h or
 * cfg; slow not 0 or 1; l1, fm, chunk or loss_cap < 1; bs < 2 or odd; 'fast' pow not 1 or 2; 'slow' l2 or nh2 < 1; world
 * < 1 or not a power of two; rank outside [0, world); no pairs, a null plane, an H or W < 1.  ADCENSUS_ELIMIT: an H or W
 * above 32767; l1 > 8; fm > 128; world above 256 or above 2 bs; 'slow' fm not a multiple of 16, l2 > 4, nh2 not 128, 256
 * or 384, or 2 bs fm ws^2 >= 2^31.  ADCENSUS_ELIMIT also when a 'fast' patch's activations exceed shared memory.
 *
 * world 1 (one GPU): the step is captured once into a CUDA graph of mccnn_trainer_launches_per_step kernels, which
 * mccnn_trainer_run and mccnn_trainer_step_patches launch.
 *
 * world >= 2 (data-parallel training): the trainer of rank `rank` of `world` ranks, each on its own device with the same
 * pair table, parameters and momenta.  A step is three segments, each a captured graph, with two all-gathers the caller
 * runs on `stream` between them: after segment 0 of SHARD_TOWER_OUT, after segment 1 of SHARD_WGRAD_PART, every rank's
 * slots (mccnn_trainer_shard_slot) from that rank.  The parameters, momenta and losses are then those of the one-GPU
 * trainer of the same arch, bit for bit, on every rank.
 * 'fast': rank r holds the batch's patches n = r, r + world, ... as its patches 0, 1, ...; mccnn_trainer_size's PATCHES,
 * TOWER and DZ are that share.
 *   segment 0: the sampler and the tower on the rank's patches; its last layer -> its slot of SHARD_TOWER_OUT;
 *   segment 1: Normalize2 / StereoJoin1 / Margin2 on the whole batch (every rank the same), the tower's backward pass on
 *              the rank's patches and its partial weight gradient (levels 128 .. world of wgrad's tree) -> its slot of
 *              SHARD_WGRAD_PART;
 *   segment 2: the tree's levels world / 2 .. 1 over the ranks' partials, then the update.
 * 'slow': the buffers are the whole batch's.  Rank r owns the patches [N r / world, N (r + 1) / world) and in each tower
 * layer the weight-gradient splits that start in them (mccnn_trainer_slow_shard_plan); it runs the tower on its patches
 * and on those its splits read past them.
 *   segment 0: the sampler and the tower forward; SHARD_TOWER_OUT is the last layer (ROWS), the rank's slot its rows;
 *   segment 1: the Linear layers, BCE and their gradients on the whole batch, the tower backward, the rank's splits of
 *              each layer's weight gradient; SHARD_WGRAD_PART is the split workspace, one slot per layer (piece);
 *   segment 2: the splits added in split order, then the update.
 * mccnn_trainer_run and _step_patches refuse a shard; get / set / size / reset_losses work as for one GPU, and
 * launches_per_step counts the kernels of the three segments. */
int mccnn_trainer_create(mccnn_trainer **h, const mccnn_trainer_config *cfg, const mccnn_train_pair *pairs, int n_pairs,
			 int device, adcensus_stream_t stream);
int mccnn_trainer_destroy(mccnn_trainer *h);

/* nsteps <= chunk training steps: warps (nsteps, N) mccnn_warp (pinned host or device; it must stay unchanged until the
 * copy has run on `stream`), then per step the sampler, forward, backward and the update with the scalar (float)(-lr).
 * Each step's loss (Margin2's mean) goes to the next entry of the loss buffer.  Asynchronous. */
int mccnn_trainer_run(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr, adcensus_stream_t stream);

/* One step from given patches ((N, 1, ws, ws) float32) instead of the sampler. */
int mccnn_trainer_step_patches(mccnn_trainer *h, const float *patches, double lr, adcensus_stream_t stream);

/* the next nsteps <= chunk steps' records of the patches the rank samples, (nsteps, its share) mccnn_warp ('fast': the
 * patches rank, rank + world, ...; 'slow': the patches plan[0] .. plan[2] - 1), and the lr; then call the segments 0,
 * 1, 2 once per step, in order */
int mccnn_trainer_shard_begin(mccnn_trainer *h, const mccnn_warp *warps, int nsteps, double lr, adcensus_stream_t stream);
int mccnn_trainer_shard_segment(mccnn_trainer *h, int segment, adcensus_stream_t stream);
/* a gathered buffer (trainer-owned device memory, *count floats), its number of pieces, and the slot of piece `piece`
 * that rank `rank` owns (offset and count in floats; a count may be 0) */
enum { MCCNN_SHARD_TOWER_OUT, MCCNN_SHARD_WGRAD_PART };
int mccnn_trainer_shard_buffer(mccnn_trainer *h, int what, float **ptr, long long *count);
int mccnn_trainer_shard_pieces(mccnn_trainer *h, int what);
int mccnn_trainer_shard_slot(mccnn_trainer *h, int what, int piece, int rank, long long *offset, long long *count);
/* HOST helper: a slow shard's share for (l1, fm, bs) -> plan (3 + 3 l1): the patches it owns [plan[0], plan[1]), the end
 * plan[2] of the patches it runs, then per layer k the splits it owns [plan[3 + 3k], plan[4 + 3k]) of plan[5 + 3k] */
int mccnn_trainer_slow_shard_plan(int l1, int fm, int bs, int rank, int world, long long *plan);

/* The trainer's buffers, for get / set (set: PARAMS and MOMENTA only) and the tests.  Sizes in floats from
 * mccnn_trainer_size.  TOWER: every layer's output, layer k (N, fm, s_k, s_k) after the previous layers, s_k = ws - 2k, post
 * ReLU except the last ('fast') or post ReLU ('slow'); DZ: the gradient of the loss wrt each layer's pre-activation output,
 * same layout; LOSS (loss_cap).
 * 'fast' only: NORM (N) = sum of squares + 1e-5; NORMALIZED (N, fm); JOIN (bs); JOIN_GRAD (bs) Margin2's gradInput /
 * (bs / 2); HINGE (bs / 2); NORM_GRAD_OUT (N, fm) the gradient wrt Normalize2's output.
 * 'slow' only: ROWS (bs, 2 fm) the reshaped rows (a view of TOWER's last layer); FC each Linear's output, the hidden ones
 * (bs, nh2) after their ReLU, then the last one's (bs) before the Sigmoid; SIGMOID (bs); BCE_GRAD (bs) the criterion's
 * gradInput; ROWS_GRAD (bs, 2 fm) the gradient arriving at the tower (wrt its last ReLU's output).
 * An id that does not apply to the handle's arch: size -1, get ADCENSUS_EINVAL. */
enum {
	MCCNN_TRAIN_PARAMS, MCCNN_TRAIN_MOMENTA, MCCNN_TRAIN_GRADS, MCCNN_TRAIN_PATCHES, MCCNN_TRAIN_TOWER, MCCNN_TRAIN_NORM,
	MCCNN_TRAIN_NORMALIZED, MCCNN_TRAIN_JOIN, MCCNN_TRAIN_JOIN_GRAD, MCCNN_TRAIN_HINGE, MCCNN_TRAIN_NORM_GRAD_OUT,
	MCCNN_TRAIN_DZ, MCCNN_TRAIN_LOSS, MCCNN_TRAIN_ROWS, MCCNN_TRAIN_FC, MCCNN_TRAIN_SIGMOID, MCCNN_TRAIN_BCE_GRAD,
	MCCNN_TRAIN_ROWS_GRAD, MCCNN_TRAIN_NBUF
};
long long mccnn_trainer_size(mccnn_trainer *h, int what);
int mccnn_trainer_get(mccnn_trainer *h, int what, float *dst, adcensus_stream_t stream);
int mccnn_trainer_set(mccnn_trainer *h, int what, const float *src, adcensus_stream_t stream);
/* the next step's loss goes to entry 0 of the loss buffer */
int mccnn_trainer_reset_losses(mccnn_trainer *h, adcensus_stream_t stream);
int mccnn_trainer_launches_per_step(mccnn_trainer *h);

/* HOST helper: the swaps i = i0 .. i0 + k - 1 of THTensor_(randperm) on perm (n) int64: swap perm[i] and
 * perm[i + draws[j] % (n - i)], draws the generator's 32-bit outputs in order (i0 + k <= n - 1). */
int mccnn_randperm_swaps(long long *perm, long long n, long long i0, const unsigned *draws, long long k);

/* HOST helper: the sample boundaries of main.lua:791-841 for dataset mb in a buffer of the generator's 32-bit outputs.
 * A sample is `base` words (the torch.uniform calls of :791-818), then light, exp, the d_exp test, exp_ only when that
 * test passes (raw / 2^32 < d_exp in double), then the d_light test: base + 4 or base + 5 words.  Walks from raw[0]
 * and writes the first word of each whole sample to starts, at most `cap` of them; *count gets their number and *used
 * the words they take (the words from *used on belong to the next sample). */
int mccnn_mb_sample_starts(const unsigned *raw, long long n_raw, int base, double d_exp, long long *starts, long long cap,
			   long long *count, long long *used);

/* ---- images of the results: samples/bin2png.lua and main.lua -debug (csrc/render.cu, render.py) ----------------------
 * Every output is 8-bit, quantised as Torch7's image.save writes a float image: clamp to [0, 1] (NaN -> 0, as x86's
 * conversion gives), times 255 in double, truncated.  Grey images are (H, W) bytes, colour images (H, W, 3) R, G, B
 * bytes, both in the PNG's pixel order.  Input maps are DEVICE float32 (H, W). */

#define ADCENSUS_ERANGE (-3)   /* mccnn_render_jet: an input whose colour-map value is NaN or outside [-0.1, 4.1] */
#define ADCENSUS_EIO (-4)      /* mccnn_render_volume_file: the file cannot be opened or is shorter than D * H * W floats */

/* bin2png.lua:17-24 for a (D, H, W) float32 little-endian volume FILE (left.bin / right.bin): NaN -> 1e38 (fromfile),
 * the 1-based arg-min over D keeping the first index on ties (TH's CPU min), divided by D in fp32, quantised into grey
 * (H, W) DEVICE bytes.  The volume is read in row chunks of at most 64 MiB through two pinned host buffers, each chunk's
 * copy overlapping the previous chunk's kernel; neither the host nor the device ever holds it whole.  Returns once the
 * file has been read; grey is complete in `stream`'s order.  D, H, W >= 1 and H * W < 2^31 (else ADCENSUS_EINVAL). */
int mccnn_render_volume_file(const char *path, int D, int H, int W, unsigned char *grey, adcensus_stream_t stream);

/* bin2png.lua:27-28: grey = quantise(f32(x) / d) with NaN -> 1e38 first (fromfile), for a map x (H, W). */
int mccnn_render_map(const float *x, int H, int W, int d, unsigned char *grey, adcensus_stream_t stream);

/* adcensus.grey2jet (adcensus.cu:2001-2053) of the map as main.lua:1242 / 1260 give it: v = ((double)x + 1) / disp_max * 4
 * in double, the five bands with the reference's comparisons, rgb (H, W, 3) = the quantised colours.  mask_blue != 0
 * multiplies the blue channel by (x != 0) before quantising (main.lua:1261, the ground-truth image).  The reference asserts
 * on a value outside the bands; here the kernel raises a device flag, the call waits for `stream` and returns
 * ADCENSUS_ERANGE (rgb is then written, with black at the refused pixels).  disp_max >= 1. */
int mccnn_render_jet(const float *x, int H, int W, int disp_max, int mask_blue, unsigned char *rgb, adcensus_stream_t stream);

/* main.lua:1243-1252 in fp32 as the cutorch ops compute it: grey = x0 * 50 + 150, then div(255), which cutorch performs as a
 * multiplication by f32(1 / 255); mask = gt != 0, bad = (|gt - pred| > err_at) * mask, good = (|gt - pred| <= err_at) * mask;
 * R = grey + 0.5 bad - 0.5 good, G = grey - 0.5 bad + 0.5 good, B = grey - 0.5 bad - 0.5 good (each term added in that
 * order), quantised into rgb (H, W, 3).  x0, pred and gt are (H, W). */
int mccnn_render_error(const float *x0, const float *pred, const float *gt, int H, int W, float err_at, unsigned char *rgb,
		       adcensus_stream_t stream);

/* ---- the KITTI 2012 / 2015 devkits' stereo metrics (csrc/kitti_eval.cu, kitti_eval.py) ---------------------------------
 * One estimate against its two PNG16 ground truths (disp_noc* and disp_occ*, uint16 disparity * 256, 0 = none) and, for
 * KITTI 2015, its obj_map (8-bit, 0 = background, else foreground), restated from the devkits' description (DESIGN.md §17;
 * parity with the devkit binaries is not pinned).
 *
 * The estimate is either a float map `disp` (quantised as dataio.write_png16 writes it: v = d < 1e-5 ? 0 : d * 256 in fp32,
 * truncated, clamped to [0, 65535], NaN -> 0) or the stored values `disp16`; exactly one of them is non-NULL.  v == 0 is
 * invalid (-1), else d = v / 256.  Then interpolateBackground: each row's interior runs of invalid pixels take the smaller
 * of their two valid neighbours, the pixels before the row's first valid pixel its value, those after its last valid pixel
 * its value; then the rows above the first row with a valid pixel take that row, those below the last such row that row;
 * whatever is left stays -1.  `ipol` (H, W) receives that map when non-NULL.
 *
 * Over the pixels with ground truth, e = |gt / 256 - ipol| in fp32; per region r (0 = noc, 1 = all, i.e. occ) the int64
 * counts[r * MCCNN_KITTI_NCOUNT + k] below, and sums[r] = sum of e in float64, reduced in a fixed order (the same bits on
 * every run).  D1 bad: e > 3 and e / (gt / 256) > 0.05f (fp32 divide).  obj_map NULL: every pixel is background.  DEVICE
 * pointers; counts and sums are overwritten.  H, W >= 1, H * W < 2^31 (else ADCENSUS_EINVAL / ADCENSUS_ELIMIT). */
enum {
	MCCNN_KITTI_GT,          /* pixels with ground truth */
	MCCNN_KITTI_DENSE,       /* ... whose estimate was valid before the interpolation (density's numerator) */
	MCCNN_KITTI_OUT2,        /* ... with e > 2 */
	MCCNN_KITTI_OUT3,        /* e > 3 */
	MCCNN_KITTI_OUT4,        /* e > 4 */
	MCCNN_KITTI_OUT5,        /* e > 5 */
	MCCNN_KITTI_D1_BG,       /* D1-bad background pixels */
	MCCNN_KITTI_D1_FG,       /* D1-bad foreground pixels */
	MCCNN_KITTI_GT_BG,       /* background pixels with ground truth */
	MCCNN_KITTI_GT_FG,       /* foreground pixels with ground truth */
	MCCNN_KITTI_NCOUNT
};
int mccnn_kitti_devkit_counts(const float *disp, const unsigned short *disp16, const unsigned short *gt_noc,
			      const unsigned short *gt_occ, const unsigned char *obj_map, int H, int W, float *ipol,
			      long long *counts, double *sums, adcensus_stream_t stream);

/* ---- the MiddEval3 SDK's evaldisp metrics (csrc/mb_eval.cu, mb_eval.py) -------------------------------------------------
 * One map `disp` (h, w) against its ground truth `gt` (Hg, Wg), top-down rows, +inf = unknown, restated from the SDK's
 * evaldisp (DESIGN.md §18; parity with the SDK binary and the website is not pinned).  scale = Wg / w must be 1, 2 or 4
 * with Wg == scale w and Hg == scale h (else ADCENSUS_EINVAL); Hg * Wg < 2^31 (else ADCENSUS_ELIMIT).
 *
 * Per gt pixel (x, y) with gt != +inf, in fp32: d = (float)scale * disp[y / scale][x / scale]; valid when d != +inf; a
 * valid d becomes max(0, min(maxd, d)) with maxd = (float)(scale * maxdisp), both as (a < b) ? a : b / (a > b) ? a : b (NaN
 * stays NaN, -inf becomes 0); err = fabsf(d - gt).  Region 0 (nonocc) takes the pixels whose `mask` (Hg, Wg) byte is 255,
 * every pixel when mask is NULL (evaldisp without a mask); region 1 (all) takes every pixel.
 *
 * Outputs, DEVICE pointers, overwritten: counts[r * MCCNN_MB_NCOUNT + k] int64; sums[2 r] = sum of err and sums[2 r + 1] =
 * sum of (double)err^2 over the valid pixels, float64 in a fixed order (the same bits on every run); quantiles[4 r + j] the
 * k-th smallest err over the valid pixels, k = ceil(q nvalid) for q = 0.50, 0.90, 0.95, 0.99 (exact, by radix select on
 * the fp32 bits; NaN errs last), NaN when there is none.  `scratch` is a DEVICE buffer of MCCNN_MB_EVAL_SCRATCH_BYTES bytes,
 * 8-byte aligned, that no other call uses until this one has run; nothing is allocated and nothing is read back.
 * maxdisp >= 1. */
#define MCCNN_MB_EVAL_SCRATCH_BYTES 49152
enum {
	MCCNN_MB_N,          /* pixels of the region with known ground truth */
	MCCNN_MB_VALID,      /* ... whose d is not +inf */
	MCCNN_MB_BAD05,      /* valid with err > 0.5 */
	MCCNN_MB_BAD1,       /* err > 1 */
	MCCNN_MB_BAD2,       /* err > 2 */
	MCCNN_MB_BAD4,       /* err > 4 */
	MCCNN_MB_INVALID,    /* ... whose d is +inf */
	MCCNN_MB_NCOUNT
};
int mccnn_mb_evaldisp(const float *disp, int h, int w, const float *gt, int Hg, int Wg, const unsigned char *mask,
		      int maxdisp, long long *counts, double *sums, float *quantiles, void *scratch,
		      adcensus_stream_t stream);

/* ---- metric depth, point clouds and depth metrics (csrc/depth.cu, depth.py; DESIGN §20) ---------------------------------
 * An addition beyond the reference.  A disparity d (H,W) at pixel (x, y) is valid when it is finite and s = d + doffs > 0
 * (fp32 add); then, each operation rounded once in fp32 and in this order, Z = fB / s, X = ((x - cx) * Z) / f,
 * Y = ((y - cy) * Z) / f, where fB is f * baseline computed in double and rounded once to float by the caller.  max_depth
 * (> 0; +inf for none) also makes Z > max_depth invalid.  Every entry checks, before any launch: H, W >= 1, f > 0, fB > 0,
 * finite f, fB, cx, cy, doffs, max_depth > 0 (else ADCENSUS_EINVAL); H * W < 2^31 (else ADCENSUS_ELIMIT).  DEVICE pointers;
 * asynchronous on `stream`.
 *
 * mccnn_disp_to_depth: Z (H,W), and X, Y (H,W) unless both are NULL; NaN at invalid pixels. */
int mccnn_disp_to_depth(const float *disp, int H, int W, float f, float cx, float cy, float fB, float doffs, float max_depth,
			float *Z, float *X, float *Y, adcensus_stream_t stream);
/* mccnn_point_cloud_count: the number of valid pixels, to count (one DEVICE int64).
 * mccnn_point_cloud_fill: one binary little-endian PLY vertex record per valid pixel, in row-major order, packed 15 bytes
 * apiece (float x, y, z; uchar red, green, blue) into out (16-byte aligned, at least 15 cap bytes); records past cap are
 * dropped.  The colour is rgb (H,W,3) R, G, B bytes (nch 3) or (H,W) grey bytes repeated three times (nch 1).  The order is
 * fixed (per-block counts, an exclusive 64-bit scan over the blocks, then the fill): the same bytes on every run. */
int mccnn_point_cloud_count(const float *disp, int H, int W, float fB, float doffs, float max_depth, long long *count,
			    adcensus_stream_t stream);
int mccnn_point_cloud_fill(const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy, float fB,
			   float doffs, float max_depth, unsigned char *out, long long cap, adcensus_stream_t stream);
/* The depth metrics of pred against the ground-truth disparity gt (H,W), both turned into depth by the rule above without
 * the cap; with pred_depth != 0, pred already holds depths in metres, valid where finite and > 0 (a depth map read back).  S = the pixels whose gt depth Zg is valid and lies in [min_depth, max_depth] (fp32 compares; 0 < min_depth <=
 * max_depth, else ADCENSUS_EINVAL).  Over S and a valid predicted depth Z, clamped to [min_depth, max_depth] in fp32, in
 * float64: sums[0] = sum |Z - Zg| / Zg, sums[1] = sum (Z - Zg)^2 / Zg, sums[2] = sum (Z - Zg)^2, sums[3] = sum (log Z -
 * log Zg)^2, each block summing a fixed range in a fixed order and one block adding the block sums in a fixed order (the
 * same bits on every run and GPU); counts (int64) as below, with r = max(Z / Zg, Zg / Z) in double. */
enum {
	MCCNN_DEPTH_GT,          /* |S| */
	MCCNN_DEPTH_N,           /* |S and a valid prediction| */
	MCCNN_DEPTH_A1,          /* ... with r < 1.25 */
	MCCNN_DEPTH_A2,          /* r < 1.25^2 */
	MCCNN_DEPTH_A3,          /* r < 1.25^3 */
	MCCNN_DEPTH_NCOUNT
};
int mccnn_depth_metrics(const float *pred, int pred_depth, const float *gt, int H, int W, float fB, float doffs, float min_depth,
			float max_depth, long long *counts, double *sums, adcensus_stream_t stream);

/* ---- LiDAR scans projected into sparse depth maps (csrc/depth.cu, depth.py; DESIGN §21) ---------------------------------
 * An addition beyond the reference.  mccnn_velo_depth_map: pts (n, 4) float32 x, y, z, reflectance (DEVICE, 16-byte
 * aligned), P the 3x4 row-major velodyne-to-image matrix (12 HOST floats, read during the call), depth (H,W) float32
 * (DEVICE).  Each point, in fp32 with every operation rounded once: x' = ((P00 x + P01 y) + P02 z) + P03, likewise y' and z'
 * from rows 1 and 2; kept when min_depth < z' < +inf; its pixel u = rint(x' / z') - 1, v = rint(y' / z') - 1 (rint: to
 * nearest, ties to even), kept inside [0, W) x [0, H).  Each pixel gets the smallest z' of its points (the smallest index
 * breaks a tie) and 0 when it has none: the same bits on every run and GPU.  Refuses a NULL or unaligned pointer, n < 0,
 * H or W < 1, min_depth < 0 or not finite, a non-finite P entry (ADCENSUS_EINVAL); H * W >= 2^31 or n >= 2^32
 * (ADCENSUS_ELIMIT).  pts may be NULL when n == 0.  Asynchronous on `stream`. */
int mccnn_velo_depth_map(const float *pts, long long n, const float *P, int H, int W, float min_depth, float *depth,
			 adcensus_stream_t stream);

/* ---- stereo rectification of calibrated raw cameras (csrc/rectify.cu, rectify.py; DESIGN §22) -------------------------
 * An addition beyond the reference.  mccnn_rectify_pair: both views of a raw pair, left and right (H,W) grey or (H,W,3)
 * R, G, B bytes (nch 1 or 3, DEVICE), rectified in one launch into out_left and out_right (Ho,Wo[,3]) bytes (DEVICE), and
 * with a non-NULL `valid` the left view's validity (Ho,Wo) bytes, 1 valid and 0 not.  params_left / params_right: the
 * MCCNN_RECTIFY_NPARAM HOST floats of each camera, read during the call: iR = inv(P[:, :3] R) row-major (computed in
 * float64 and rounded once to fp32), fx, fy, cx, cy of K, then k1 k2 p1 p2 k3 k4 k5 k6 (missing ones 0).
 * Output pixel (u, v), in fp32 with every operation rounded once, in this order (OpenCV's initUndistortRectifyMap model):
 *   X = (iR00 u + iR01 v) + iR02, Y and Z likewise from rows 1 and 2;  x = X / Z, y = Y / Z;  r2 = x x + y y;
 *   rad = (1 + r2 (k1 + r2 (k2 + r2 k3))) / (1 + r2 (k4 + r2 (k5 + r2 k6)));
 *   xd = x rad + (2 p1 x y + p2 (r2 + 2 x x));  yd = y rad + (p1 (r2 + 2 y y) + 2 p2 x y)  (products left to right);
 *   sx = fx xd + cx, sy = fy yd + cy.
 * Sampling: x0 = floor(sx), a = sx - x0, y0 = floor(sy), b = sy - y0; the taps x0, x0 + 1, y0, y0 + 1 clamped into the raw
 * image (the border replicated); v = (1 - b) ((1 - a) I00 + a I01) + b ((1 - a) I10 + a I11), the byte rint(v) (ties to
 * even), the colour channels sharing the weights.  Valid: -0.5 <= sx < W - 0.5 and -0.5 <= sy < H - 0.5.  Where Z <= 0 or
 * sx or sy is not finite the pixel is invalid and its bytes are 0.  The same bytes on every run and GPU.
 * Refuses, before any launch: a NULL pointer (valid excepted), an output overlapping an input or another output, nch not 1
 * or 3, a non-finite parameter, H, W, Ho or Wo < 1 (ADCENSUS_EINVAL); H W nch or Ho Wo nch >= 2^31 (ADCENSUS_ELIMIT).
 * Asynchronous on `stream`. */
#define MCCNN_RECTIFY_NPARAM 21
int mccnn_rectify_pair(const unsigned char *left, const unsigned char *right, int nch, int H, int W, const float *params_left,
		       const float *params_right, int Ho, int Wo, unsigned char *out_left, unsigned char *out_right,
		       unsigned char *valid, adcensus_stream_t stream);

/* ---- posed frames fused into one world-frame voxel map (csrc/fusion.cu, fusion.py; DESIGN §23) ------------------------
 * An addition beyond the reference.  A table of voxels of edge `voxel` metres, each holding n_pix (int64), n_frames (the
 * frames that put a pixel in it, int64), three float64 sums of world points and three int64 sums of colour bytes.
 * mccnn_fusion_create: an empty table on CUDA device `device`; refuses voxel not finite or <= 0 and a device that does
 * not exist (ADCENSUS_EINVAL).  Every other call makes that device current for its duration.
 * mccnn_fusion_add: one frame.  disp (H,W) float32 and rgb (H,W[,3]) bytes (nch 1 or 3) are DEVICE; f, cx, cy, fB, doffs
 * and max_depth as mccnn_point_cloud_fill; pose12 the 12 HOST float64 of a row-major [R | t] taking the frame's camera
 * point into the world, read during the call.  A pixel valid under §20's rule has the camera point (X, Y, Z) of its
 * point-cloud vertex and the world point w_k = ((R_k0 X + R_k1 Y) + R_k2 Z) + t_k in float64, each operation rounded once;
 * its voxel index is floor(w / voxel) (float64 division) per axis.  When each index lies in [-2^20, 2^20) its key is
 * ((ix + 2^20) << 42) | ((iy + 2^20) << 21) | (iz + 2^20), else it counts as outside and is dropped.  Each voxel's partial
 * starts at +0.0 and adds its pixels in row-major order; the table's sum starts at +0.0 and adds the frames' partials in
 * the order they were added.  stats (3 DEVICE int64) receives the frame's pixels in the table, its pixels outside the key
 * range and the table's voxel count afterwards.  One int64 is read back (the stream is synchronised) to size the table,
 * which grows by reallocation.  Refuses NULL pointers, nch not 1 or 3, H or W < 1, a camera as mccnn_point_cloud_fill
 * refuses, a non-finite pose entry (ADCENSUS_EINVAL) and H W nch >= 2^31 (ADCENSUS_ELIMIT), before any launch.
 * mccnn_fusion_size: the voxel count (-1 for NULL).
 * mccnn_fusion_count: the voxels with n_frames >= min_frames (min_frames >= 1), to count (one DEVICE int64).
 * mccnn_fusion_fill: one 15-byte PLY vertex record per such voxel in ascending key order (records past cap are dropped):
 * the position float32(sum / n_pix) per axis, divided in float64, and the colour (C + n_pix / 2) / n_pix per channel in
 * integers.  Blocks count their voxels, one block scans the counts in block order (64-bit), then the fill: the same bytes
 * on every run and GPU.
 * mccnn_fusion_table: the table in ascending key order into DEVICE arrays of mccnn_fusion_size entries: keys, npix,
 * nframes, and sums and colours as three planes (x, y, z / r, g, b) of that many entries each.
 * All asynchronous on `stream` except the read-back of mccnn_fusion_add. */
typedef struct mccnn_fusion mccnn_fusion;
int mccnn_fusion_create(mccnn_fusion **out, double voxel, int device);
int mccnn_fusion_add(mccnn_fusion *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy,
		     float fB, float doffs, float max_depth, const double *pose12, long long *stats, adcensus_stream_t stream);
long long mccnn_fusion_size(const mccnn_fusion *h);
int mccnn_fusion_count(const mccnn_fusion *h, int min_frames, long long *count, adcensus_stream_t stream);
int mccnn_fusion_fill(const mccnn_fusion *h, int min_frames, unsigned char *out, long long cap, adcensus_stream_t stream);
int mccnn_fusion_table(const mccnn_fusion *h, unsigned long long *keys, long long *npix, long long *nframes, double *sums,
		       long long *colours, adcensus_stream_t stream);
void mccnn_fusion_destroy(mccnn_fusion *h);

/* ---- posed frames fused into a truncated signed distance field (csrc/tsdf.cu, fusion.py; DESIGN §24) -------------------
 * An addition beyond the reference.  A table of bricks of 8^3 voxels of edge `voxel` metres, truncation `trunc` metres.
 * A brick's key is §23's key of its index floor(i / 8), i = floor(w / voxel) the voxel index; each voxel holds S (float64),
 * n (the frames that updated it), nc and three colour byte sums (int32): MCCNN_TSDF_BRICK_BYTES per brick.
 * mccnn_tsdf_create: an empty field on CUDA device `device`; refuses voxel not finite or <= 0, trunc not finite or < voxel
 * and a device that does not exist (ADCENSUS_EINVAL), and ceil(trunc / (4 voxel)) > 64 (ADCENSUS_ELIMIT).
 * mccnn_tsdf_add: one frame, its arguments as mccnn_fusion_add's.  With K = ceil(trunc / (4 voxel)) and s = fp32(trunc / K),
 * each valid pixel of depth Z allocates the bricks of its ray points at z = Z + fp32(j) s (fp32), j = -K .. K, z > 0,
 * placed as fusion places a pixel; points whose brick lies outside [-2^20, 2^20) on some axis are counted.  Then every
 * voxel of every brick: centre c = (i + 0.5) voxel, q = R^T (c - t) in float64 (((R_0a d_0 + R_1a d_1) + R_2a d_2), d =
 * c - t), skipped unless q_z > 0 and the pixel (floor((q_x / q_z) f + cx + 0.5), likewise y) lies in the image and has a
 * depth Z; eta = Z - q_z; skipped when eta < -trunc; else S += min(eta, trunc) / trunc, n += 1, and when |eta| < trunc the
 * pixel's colour bytes are added and nc += 1.  stats (2 DEVICE int64) receives the frame's valid pixels and its points
 * outside the key range.  One int64 is read back (the stream is synchronised).  Refuses what mccnn_fusion_add refuses,
 * and (ADCENSUS_ELIMIT) H W (2K + 1) >= 2^31 and a frame beyond the 2^23-th.
 * mccnn_tsdf_bricks: the brick count (-1 for NULL).  mccnn_tsdf_pool_bytes: the bytes the brick pool holds (-1 for NULL).
 * mccnn_tsdf_table: the field in ascending key order into DEVICE arrays: keys (bricks), then per voxel (brick, z, y, x):
 * S, n, nc (bricks 512 each) and colours (bricks 512 3, r g b interleaved).
 * mccnn_tsdf_mesh_count: the vertex and face counts (2 DEVICE int64) of the mesh of the voxels with n >= min_frames.
 * mccnn_tsdf_mesh_fill: its 15-byte PLY vertex records (vertices past vcap dropped; vcap < 2^31) and int32 faces (3 per
 * face, faces past fcap dropped): marching tetrahedra on the Kuhn split, DESIGN §24's order and orientation.
 * mccnn_tsdf_render: the (H,W) DEVICE float32 depth map seen from pose12 under f, cx, cy: the first zero crossing, from
 * positive to negative, of the trilinear field sampled at camera depths fp32(k voxel), k >= 1, up to max_depth (may be
 * +inf); NaN where none.  The brick bounds are read back (the stream is synchronised).  Refuses min_frames < 1, H or W < 1,
 * a bad camera or pose and, with max_depth +inf, a singular R (ADCENSUS_EINVAL).
 * All asynchronous on `stream` except the read-backs named. */
#define MCCNN_TSDF_BRICK_BYTES 14336
typedef struct mccnn_tsdf mccnn_tsdf;
int mccnn_tsdf_create(mccnn_tsdf **out, double voxel, double trunc, int device);
int mccnn_tsdf_add(mccnn_tsdf *h, const float *disp, const unsigned char *rgb, int nch, int H, int W, float f, float cx, float cy,
		   float fB, float doffs, float max_depth, const double *pose12, long long *stats, adcensus_stream_t stream);
long long mccnn_tsdf_bricks(const mccnn_tsdf *h);
long long mccnn_tsdf_pool_bytes(const mccnn_tsdf *h);
int mccnn_tsdf_table(const mccnn_tsdf *h, unsigned long long *keys, double *S, int *n, int *nc, int *colours, adcensus_stream_t stream);
int mccnn_tsdf_mesh_count(const mccnn_tsdf *h, int min_frames, long long *counts, adcensus_stream_t stream);
int mccnn_tsdf_mesh_fill(const mccnn_tsdf *h, int min_frames, unsigned char *verts, long long vcap, int *faces, long long fcap,
			 adcensus_stream_t stream);
int mccnn_tsdf_render(const mccnn_tsdf *h, int min_frames, int H, int W, float f, float cx, float cy, float max_depth,
		      const double *pose12, float *depth, adcensus_stream_t stream);
void mccnn_tsdf_destroy(mccnn_tsdf *h);

/* ---- frame-to-model tracking against the distance field (csrc/track.cu, track.py; DESIGN §25) ------------------------
 * An addition beyond the reference.  A handle owns two pyramids of MCCNN_TRACK_LEVELS levels at one (H, W): the source
 * (a frame's disparity) and the model (a depth map TSDF.render returned).  Level l keeps the full-resolution pixels
 * (2^l x, 2^l y) and is ceil(H / 2^l) x ceil(W / 2^l); each pixel has a float64 vertex (the fp32 camera.cuh bits of §20's
 * rule) and a float64 normal, NaN where there is none.
 * mccnn_track_create: refuses H or W < 1 and a device that does not exist (ADCENSUS_EINVAL), H W >= 2^31 (ADCENSUS_ELIMIT).
 * mccnn_track_source: the source pyramid of the DEVICE (H,W) disparity map under a camera as mccnn_tsdf_add takes it.
 * mccnn_track_model: the model pyramid of the DEVICE (H,W) depth map `depth` (NaN = no vertex) under f, cx, cy; the step
 * projects into the model with this camera.
 * mccnn_track_step: one projective point-to-plane ICP reduce at `level` for the source-to-model pose pose12 ([R | t]):
 * sums (28 host float64) receives the upper triangle of J^T J row by row, J^T r and r^2 over the inlier pixels, summed in
 * DESIGN §25's fixed tree.  With gates = {g_min, rho} (host), the photometric term of each pixel (DESIGN §26) is reduced
 * in the same pass and tree: sums (56 host float64) then receives those 28 geometric sums, bit for bit the gate-less
 * step's, followed by the 28 photometric ones.  counts (3 host int64) gets the geometric inliers, the photometric
 * inliers (0 without gates) and the level's source vertices.  One device-to-host copy; the stream is synchronised.
 * Refuses (ADCENSUS_EINVAL) a level outside [0, MCCNN_TRACK_LEVELS), a non-finite pose, delta not finite or <= 0,
 * cos_theta outside [-1, 1], NULL outputs and a handle without both pyramids; with gates also g_min or rho not finite or
 * < 0 and a handle without both intensity pyramids.
 * mccnn_track_maps: a level's vertices and normals (`which` 0 source, 1 model) into two DEVICE arrays of 3 planes (x, y,
 * z) of ceil(H / 2^l) ceil(W / 2^l) float64 each.
 * Every argument is checked before any launch; all asynchronous on `stream` except the step's read-back. */
#define MCCNN_TRACK_LEVELS 3
#define MCCNN_TRACK_SUMS 28
typedef struct mccnn_track mccnn_track;
int mccnn_track_create(mccnn_track **out, int H, int W, int device);
int mccnn_track_source(mccnn_track *h, const float *disp, float f, float cx, float cy, float fB, float doffs, float max_depth,
		       adcensus_stream_t stream);
int mccnn_track_model(mccnn_track *h, const float *depth, float f, float cx, float cy, adcensus_stream_t stream);
int mccnn_track_step(mccnn_track *h, int level, const double *pose12, double delta, double cos_theta, const double *gates,
		     double *sums, long long *counts, adcensus_stream_t stream);
int mccnn_track_maps(const mccnn_track *h, int which, int level, double *vertices, double *normals, adcensus_stream_t stream);
/* The photometric term's pyramids (DESIGN §26).  Their memory is allocated by the first mccnn_track_intensity; a tracker
 * that never uses them keeps only the step's 28 rows of photometric chunk sums more.
 * mccnn_track_intensity: the intensity pyramid of the DEVICE (H,W) grey (nch 1) or (H,W,3) R, G, B (nch 3) byte image
 * `img`: `which` 0 the source (the frame's left image), 1 the reference (the left image of the frame the model was
 * rendered at), which also gets its g_x and g_y planes.  Refuses which outside {0, 1} and nch outside {1, 3}.
 * mccnn_track_intensity_maps: a level's intensities (ceil(H / 2^l) ceil(W / 2^l) float32) into the DEVICE array I, and for
 * the reference its g_x and g_y (float64 each, NaN on the level's border) into gx and gy, which must be NULL for the
 * source. */
int mccnn_track_intensity(mccnn_track *h, int which, const unsigned char *img, int nch, adcensus_stream_t stream);
int mccnn_track_intensity_maps(const mccnn_track *h, int which, int level, float *I, double *gx, double *gy,
			       adcensus_stream_t stream);
void mccnn_track_destroy(mccnn_track *h);

#ifdef __cplusplus
}
#endif
#endif
