// camera.cuh -- the per-pixel depth rule of DESIGN §20, shared by depth.cu (depth maps, point clouds) and fusion.cu (the
// world-frame map of §23), so a fused point is the same fp32 camera point as its point-cloud vertex.
#pragma once

#include <math.h>

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
