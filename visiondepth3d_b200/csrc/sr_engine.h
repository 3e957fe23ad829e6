// sr_engine.h -- what vd3d_api.cu's vd3d_sr_upscale uses of the SR engine container (depth_engine.cu)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/vd3d.h"

namespace vd3d {
// the stream the engine enqueues on (vd3d_sr_create's argument)
cudaStream_t sr_stream(vd3d_depth* e);
// a named device buffer of the engine, grown to at least `bytes`
int sr_buffer(vd3d_depth* e, const char* name, size_t bytes, void** out);
// k_sr_in + the conv stack of vd3d_sr_forward on the network input BGR u8 [h,w,3] (device); *conv receives the last
// conv's f32 NHWC output [h*w, 48].  Enqueued on the engine stream; counts its launches on the engine.
int sr_network(vd3d_depth* e, const uint8_t* frame_dev, int h, int w, int num_conv, const float** conv);
// the network scale of an RRDBNet engine (vd3d_sr_set_rrdb), 0 for SRVGGNetCompact
int sr_net_scale(vd3d_depth* e);
// k_sr_in + the RRDBNet of an RRDBNet engine on BGR u8 [h,w,3] (device); *rgb receives its f32 output
// [scale h * scale w, 32] (RGB in columns 0..2).  Enqueued on the engine stream.
int rrdb_network(vd3d_depth* e, const uint8_t* frame_dev, int h, int w, const float** rgb);
}  // namespace vd3d
