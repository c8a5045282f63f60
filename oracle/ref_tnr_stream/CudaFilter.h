// oracle/ref_tnr_stream/CudaFilter.h -- TEST INFRASTRUCTURE ONLY.
// Stand-in for the reference's CudaFilter.h (included by VideoFilter.hpp:7, not in the reference tree): the four cudaTNR*
// calls CudaTemporalNRFilter makes (:214-267), mapped one to one onto amtk_tnr_stream_* of include/amtk_b200.h.  This is
// the mapping INTEGRATION.md section 5c documents.  Included by oracle/ref_tnr_stream_glue.cpp after its AVFrame stand-ins,
// which provide AVFrame, av_frame_get_buffer, av_frame_unref and bits_of(format).
#pragma once
#include <vector>

#include "../../include/amtk_b200.h"

// The library's entry points, resolved by the glue from the path the test hands it.
struct AmtkApi {
  amtk_ctx* ctx = nullptr;
  int (*stream_create)(amtk_ctx*, const amtk_tnr_params*, int, int, amtk_tnr_stream**) = nullptr;
  void (*stream_destroy)(amtk_tnr_stream*) = nullptr;
  int (*stream_send)(amtk_tnr_stream*, const amtk_clip*, int32_t) = nullptr;
  int (*stream_recv)(amtk_tnr_stream*, const amtk_clip*, int32_t*, int*) = nullptr;
  int (*stream_finish)(amtk_tnr_stream*) = nullptr;
};
static AmtkApi g_amtk;

struct CudaTNRFilterImpl {
  amtk_tnr_stream* s = nullptr;
  int format = 0, width = 0, height = 0;      // of the first frame sent: what a received frame is allocated as
  int32_t next_tag = 0;                       // the reference's queue pairs outputs with inputs in order (:235-240)
};
typedef CudaTNRFilterImpl* CudaTNRFilter;

// The reference's filter never destroys its handle (it has no destructor); the run that created them does.
static std::vector<CudaTNRFilter> g_tnr_handles;

// One AVFrame as a one-frame amtk_clip: the planes where FFmpeg put them, host memory.
static amtk_clip clip_of(const AVFrame* f) {
  amtk_clip c = {};
  const int bits = bits_of(f->format);
  c.base = f->data[0];
  c.off_u = f->data[1] - f->data[0];
  c.off_v = f->data[2] - f->data[0];
  c.width = f->width; c.height = f->height;
  c.pitch_y = f->linesize[0]; c.pitch_uv = f->linesize[1];
  c.log_uvx = c.log_uvy = 1;
  c.bytes_per_sample = bits > 8 ? 2 : 1; c.bits_per_sample = bits;
  c.frame_stride = 0; c.num_frames = 1; c.on_device = 0;
  return c;
}

// cudaTNRCreate(temporalDistance, threshold, batchSize, interlaced) -> amtk_tnr_stream_create, every frame emitted
static CudaTNRFilter cudaTNRCreate(int temporalDistance, int threshold, int batchSize, int interlaced) {
  amtk_tnr_params p = { temporalDistance, threshold, interlaced ? 1 : 0 };
  amtk_tnr_stream* s = nullptr;
  if (!g_amtk.stream_create(g_amtk.ctx, &p, batchSize, 0, &s)) return nullptr;
  CudaTNRFilter f = new CudaTNRFilterImpl();
  f->s = s;
  g_tnr_handles.push_back(f);
  return f;
}

// cudaTNRSendFrame -> amtk_tnr_stream_send; 0 on success
static int cudaTNRSendFrame(CudaTNRFilter f, AVFrame* frame) {
  if (f->next_tag == 0) { f->format = frame->format; f->width = frame->width; f->height = frame->height; }
  const amtk_clip c = clip_of(frame);
  return g_amtk.stream_send(f->s, &c, f->next_tag++) ? 0 : -1;
}

// cudaTNRRecvFrame -> amtk_tnr_stream_recv into a freshly allocated frame; 0 when a frame was received
static int cudaTNRRecvFrame(CudaTNRFilter f, AVFrame* frame) {
  av_frame_unref(frame);              // like FFmpeg's receive calls: copies made earlier keep their own buffer
  frame->format = f->format; frame->width = f->width; frame->height = f->height;
  if (av_frame_get_buffer(frame, 64) != 0) return -1;
  const amtk_clip c = clip_of(frame);
  int32_t tag = -1;
  int got = 0;
  if (!g_amtk.stream_recv(f->s, &c, &tag, &got)) return -1;
  if (!got) { av_frame_unref(frame); return 1; }
  return 0;
}

// cudaTNRFinish -> amtk_tnr_stream_finish; 0 on success
static int cudaTNRFinish(CudaTNRFilter f) { return g_amtk.stream_finish(f->s) ? 0 : -1; }
