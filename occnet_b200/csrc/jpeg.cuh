// Baseline JPEG decoding on the device (jpeg.cu), shared by the occb200_jpeg_* entries and the frame engine's input dtype 4.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct occb200_jpeg;

namespace occ {

// Host only, no CUDA call: parse the n files' headers and build their tables into the decoder's host state.  Every file must
// be a baseline YCbCr 4:2:0 / 4:4:4 JPEG the decoder supports (error 1 naming what is not), and want_h x want_w when
// want_h > 0.
int jpeg_prepare(occb200_jpeg* d, int n, const void* const* data, const int64_t* size, int want_h, int want_w);
// bytes of the decoded images of the last jpeg_prepare: sum of h * w * 3
int64_t jpeg_out_bytes(const occb200_jpeg* d);
// Pack the prepared files into the decoder's pinned staging buffer (after its previous upload has left it) and upload them on
// `copy`; `st` (the stream that decodes) waits for the upload.
int jpeg_upload(occb200_jpeg* d, cudaStream_t copy, cudaStream_t st);
// Decode the uploaded files on `st` into out (image i at the sum of the earlier images' h * w * 3 bytes), after clearing the
// status word; then copy the status word to the decoder's pinned host word on `st`.  kJpegLaunches kernels.
int jpeg_decode(occb200_jpeg* d, uint8_t* out, cudaStream_t st);
constexpr int kJpegLaunches = 3;
// The pinned copy of the status word of the last decode (valid once `st` has reached it): bit i % 32 set = image i was corrupt.
int jpeg_status_host(const occb200_jpeg* d);

}  // namespace occ
