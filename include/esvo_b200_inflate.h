/*
 * esvo_b200_inflate.h -- C ABI of the chunk inflater: the bz2 and LZ4 chunks of a compressed ROS1 bag (rosbag record -j,
 * rosbag record --lz4, rosbag compress) decompressed on the device.  esvo_b200.h includes this header.
 *
 * Kept apart from esvo_b200.h (as esvo_b200_bag.h): there is no oracle counterpart.  The reference is the format itself --
 * Python's bz2 (libbz2) for bz2, the LZ4 frame format v1.6 for LZ4 -- and the outputs are byte-identical to it.
 *
 * The inflater needs no esvo_ctx: the rig comes from CameraInfo messages that may themselves lie in compressed chunks, so a
 * bag is inflated before any context exists (include/esvo_b200/rosbag_events.hpp, RosBag(path, inflate_device)).
 *
 * Codecs:
 *   ESVO_CODEC_BZ2  one bzip2 stream (BZh1..BZh9), decoded completely and checked as libbz2 checks it: block sizes,
 *                   origPtr, code lengths, runs and MTF indices, every block CRC, the end-of-stream magic and the combined
 *                   CRC; after the end-of-stream marker only its zero padding may follow.  Refused as unsupported: a
 *                   randomised block (bzip2 < 0.9.5) and a stream of more than dst_size / 32768 + 4 blocks (a bzip2
 *                   compressor fills every block but the last with at least 100 000 bytes).
 *   ESVO_CODEC_LZ4  one LZ4 frame: independent or linked blocks, block checksums, content size and content checksum
 *                   (each xxHash32, verified when present), block sizes 64 KiB to 4 MiB, uncompressed blocks.  Refused as
 *                   unsupported: a dictionary ID, legacy and skippable frames.
 * Every other defect (a match before the start of the output, a write past the block or chunk size, a truncated stream,
 * a wrong checksum or CRC, an output length other than dst_size) refuses the chunk with ESVO_ERR_INVALID_ARG.
 */
#ifndef ESVO_B200_INFLATE_H_
#define ESVO_B200_INFLATE_H_

#include "esvo_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct esvo_inflater esvo_inflater;

enum { ESVO_CODEC_BZ2 = 1, ESVO_CODEC_LZ4 = 2 };

typedef struct {
  const uint8_t* src; uint64_t src_size;   /* the chunk record's data, host memory (e.g. the mapped bag) */
  uint8_t* dst;       uint64_t dst_size;   /* the chunk header's `size`; exactly that many bytes are written */
  int32_t codec;      int32_t status;      /* status: per-chunk result (ESVO_OK or the refusal's code) */
} esvo_chunk;

/* An inflater on `device` with a stream, pinned staging and scratch_bytes of device memory.  ESVO_ERR_NO_DEVICE without a
 * CUDA device (there is no CPU fallback), ESVO_ERR_CUDA when the memory cannot be had.  One inflater is not thread-safe;
 * separate inflaters are independent. */
ESVO_API int esvo_inflater_create(int device, size_t scratch_bytes, esvo_inflater** out);
ESVO_API void esvo_inflater_destroy(esvo_inflater* inf);
/* The message of the last failing call: it names the first failing chunk's index and the reason. */
ESVO_API const char* esvo_inflater_last_error(const esvo_inflater* inf);

/* Inflates chunks[0, n): packs them into batches that fit the scratch (compressed input, work buffers, output), uploads
 * each batch in one copy, inflates it and downloads the outputs.  Returns when every dst is written.  Every chunk's status
 * is set; the return value is the first failing chunk's code (ESVO_OK when none fails), and the other chunks' outputs are
 * still written.  ESVO_ERR_CAPACITY for a chunk that does not fit the scratch even alone (the message names the bytes it
 * needs); ESVO_ERR_INVALID_ARG / ESVO_ERR_UNSUPPORTED for a refused stream (see above). */
ESVO_API int esvo_inflate_chunks(esvo_inflater* inf, esvo_chunk* chunks, int n);

#ifdef __cplusplus
}
#endif
#endif /* ESVO_B200_INFLATE_H_ */
