// camera.cuh -- the per-pixel depth rule of DESIGN §20, shared by depth.cu (depth maps, point clouds), fusion.cu (the
// world-frame map of §23) and tsdf.cu (the distance field of §24), so a fused point is the same fp32 camera point as its
// point-cloud vertex; and §23's camera-to-world transform, shared by fusion.cu and tsdf.cu.
#pragma once

#include <math.h>

#include "common.cuh"

struct Cam {
	float f, cx, cy, fB, doffs, max_depth;
};

// Z of disparity d, or false when d has no depth (not finite, d + doffs <= 0, Z > max_depth)
__device__ __forceinline__ bool depth_of(float d, const Cam &c, float *z)
{
	const float s = __fadd_rn(d, c.doffs);
	if (!(isfinite(d) && s > 0.f)) return false;
	*z = __fdiv_rn(c.fB, s);
	return *z <= c.max_depth;
}

// X (u = x, c0 = cx) or Y (u = y, c0 = cy): ((u - c0) * z) / f, each operation rounded once
__device__ __forceinline__ float lateral(int u, float c0, float z, float f) { return __fdiv_rn(__fmul_rn(__fsub_rn((float)u, c0), z), f); }

struct Pose {
	double r[12];  // row-major [R | t]
};

// w = R (X, Y, Z) + t in float64, each operation rounded once and no FMA: w_k = ((R_k0 X + R_k1 Y) + R_k2 Z) + t_k
__device__ __forceinline__ void to_world(double X, double Y, double Z, const Pose &T, double *w)
{
#pragma unroll
	for (int a = 0; a < 3; a++) {
		const double *r = T.r + 4 * a;
		w[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], X), __dmul_rn(r[1], Y)), __dmul_rn(r[2], Z)), r[3]);
	}
}

// the 12 host float64 of a pose, refused (ADCENSUS_EINVAL) when NULL or not finite
inline int check_pose(const double *pose12, Pose *T)
{
	if (!pose12) return ADCENSUS_EINVAL;
	for (int k = 0; k < 12; k++) {
		if (!isfinite(pose12[k])) return ADCENSUS_EINVAL;
		T->r[k] = pose12[k];
	}
	return 0;
}
