// The screen mean of one 3D point in one view, as the projection forms a Gaussian's mean: shared by the flow plane (flow.cu)
// and point visibility (visibility.cu), so that both agree with the renderer for every camera model without a copy of them.
#pragma once
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

// the view's screen mean (px, py) of p in pixels (the projection's expressions for the view's model), and whether p passes the
// projection's cull of a mean.  The view-space depth t.z is xform4x3(p, c.viewmatrix).z, as here.
__device__ __forceinline__ bool flow_mean(const FlowCam& c, const V3& p, float& px, float& py)
{
	const V3 t = xform4x3(p, c.viewmatrix);
	if (c.model == 0 || c.model == 1) {
		const float4 h = xform4x4(p, c.projmatrix);
		const float w = 1.0f / (h.w + 0.0000001f);
		px = ndc2pix(h.x * w, c.W); py = ndc2pix(h.y * w, c.H);
		return t.z > NEAR_Z;
	}
	px = py = 0.f;
	if (t.z <= NEAR_Z) return false;
	const float tanx = c.tan_fov ? c.tan_fov[0] : c.tan_fovx, tany = c.tan_fov ? c.tan_fov[1] : c.tan_fovy;
	const float fx = c.W / (2.0f * tanx), fy = c.H / (2.0f * tany);
	if (c.model == 2) {
		const FisheyeRadial fr = fisheye_radial<false>(t.x, t.y, t.z, c.fe_k);
		if (fr.theta > c.theta_max) return false;
		px = fx * fr.a * t.x + c.cx; py = fy * fr.a * t.y + c.cy;
		return true;
	}
	const float iz = 1.0f / t.z;
	const DistTerms ds = distortion_terms<false>(t.x * iz, t.y * iz, c.dc_k);
	if (ds.r2 > c.r2_max || fmaf(-ds.d01, ds.d01, ds.d00 * ds.d11) <= 0.f) return false;
	px = fx * ds.xd + c.cx; py = fy * ds.yd + c.cy;
	return true;
}

}  // namespace mgs
