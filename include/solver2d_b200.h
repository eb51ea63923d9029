// solver2d-b200 — extensions to the solver2d C API that only make sense for the GPU library.
// A client that sticks to include/solver2d/solver2d.h never needs this header.
#pragma once

#include "s2b_device.h"
#include "solver2d/id.h"
#include "solver2d/types.h"

#ifdef __cplusplus
extern "C"
{
#endif

// The device world behind a public world id, for the stage-level entry points of s2b_device.h (schedule selection,
// counters, NCCL packing). The handle is owned by the world.
S2B_API s2bWorld* s2World_GetDevice(s2WorldId worldId);

// Bounce contacts by their shapes' restitution (default off: restitution is ignored, as in the reference). A contact's
// restitution is the larger of its two shapes' s2ShapeDef.restitution. Takes effect at the next s2World_Step.
S2B_API void s2World_EnableRestitution(s2WorldId worldId, bool enable);
// Approach speed (m/s) below which a contact does not bounce. Default 1 m/s, the reference's world->restitutionThreshold.
// A threshold that is not finite or is negative is rejected (the world keeps its threshold). Takes effect at the next
// s2World_Step.
S2B_API void s2World_SetRestitutionThreshold(s2WorldId worldId, float threshold);

// Push every pending host-side edit to the device now (s2World_Step does this itself).
S2B_API void s2World_Flush(s2WorldId worldId);

// Bulk forms of the per-body calls, for clients that touch every body every frame (one FFI call instead of Nb):
//   s2World_ApplyForcesToCenters == s2Body_ApplyForceToCenter for bodyIndices[i] with force (forcesXY[2i], forcesXY[2i+1]);
//   s2World_GetBodyTransforms    == s2Body_GetPosition + rotation for every body slot: {origin.x, origin.y, rot.s, rot.c}
//                                   into out[4 * capacity]; returns the body capacity.
S2B_API void s2World_ApplyForcesToCenters(s2WorldId worldId, const int32_t* bodyIndices, const float* forcesXY, int32_t count);
S2B_API int32_t s2World_GetBodyTransforms(s2WorldId worldId, float* out, int32_t capacity);

// Run `steps` calls of s2World_Step back to back and return the summed device time of the steps in milliseconds, each
// step bracketed by CUDA events on the world's stream. With flushL2 != 0 the L2 (50 MB on an H100) is evicted between steps
// (outside the timed intervals) so every step starts from HBM.
S2B_API float s2World_TimedSteps(s2WorldId worldId, int32_t steps, float timeStep, int32_t velIters, int32_t posIters,
								 bool warmStart, int32_t flushL2);

// The float atan2 the device kernels use (include/solver2d/atan2_f32.h), evaluated on the host: lets a CPU-only test
// pin it to the C library's atan2f.
S2B_API float s2Atan2Device(float y, float x);

#ifdef __cplusplus
}
#endif
