/*
 * esvo_b200_hotpix.h -- C ABI of hot-pixel removal at the packed event ingest: count each pixel's dvs_msgs/Event wire records,
 * select the hot pixels, and drop their events in esvo_ts_push_event_array(_dev).  esvo_b200.h includes this header.
 *
 * Replaces step 4 of the reference's data preparation (events_repacking_helper/README.md, "Remove hot pixels"), which rewrites
 * the bag with an external ROS tool.  There is no oracle counterpart (see esvo_b200_bag.h): the rule below is the
 * specification, and tests/test_gpu_hot_pixels.py holds it against numpy.
 *
 * The rule, per camera (W x H sensor, N = W * H):
 *   c[p]  number of counted records with x < W && y < H at p = y * W + x (u32); records outside the image are neither counted
 *         nor ever dropped;
 *   S1 = sum c, S2 = sum c^2 as exact integers, each converted once to double (round to nearest);
 *   mu = S1 / N;  sigma = sqrt(max(0, S2 / N - mu * mu));  p is hot iff (double)c[p] > mu + k * sigma,
 * in IEEE double, in this order, without contraction.  Every pixel counts, including pixels without events.
 */
#ifndef ESVO_B200_HOTPIX_H_
#define ESVO_B200_HOTPIX_H_

#include "esvo_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Adds the records of the runs to camera cam's counts (runs and n_events as esvo_ts_push_event_array).  The runs are copied
 * through the camera's pinned staging block, a piece at a time, so a whole recording can be counted in one call; they may be
 * reused on return.  Counts accumulate over calls until esvo_hotpix_clear. */
ESVO_API int esvo_hotpix_count_event_array(esvo_ctx* ctx, int cam, const uint8_t* const* runs, const size_t* n_events,
                                           int n_runs);
/* The same on n records already in device memory at packed_dev (any byte alignment); enqueued on the camera's stream. */
ESVO_API int esvo_hotpix_count_event_array_dev(esvo_ctx* ctx, int cam, const uint8_t* packed_dev, size_t n);

/* Computes camera cam's mask from its counts with the rule above and installs it; *n_hot (may be NULL) = the number of hot
 * pixels.  Synchronises the camera's stream once.  While a mask with at least one hot pixel is installed,
 * esvo_ts_push_event_array and esvo_ts_push_event_array_dev drop the records at its pixels before they reach the log: each
 * such push reads back the number kept and the last kept stamp (one synchronisation), and everything after the filter -- push
 * indices, order check (against the previous kept record), unordered mode, fold, refusals -- is that of a push of the kept
 * records.  One exception: the half-log refusal (ESVO_ERR_CAPACITY) applies to the records handed in, before the filter.
 * The SoA pushes (esvo_ts_push_events, _dev) are not filtered.  esvo_ts_reset keeps the mask (a log reset is not a change of
 * sensor).
 * ESVO_ERR_INVALID_ARG for k negative, NaN or infinite; ESVO_ERR_CAPACITY when a count passed 2^32 - 1 (the counts are refused
 * rather than wrapped; the installed mask is left as it was).  Both leave everything unchanged. */
ESVO_API int esvo_hotpix_select(esvo_ctx* ctx, int cam, double k, int64_t* n_hot);

/* Camera cam's counts (W*H u32) and mask (W*H u8, 1 = hot; all 0 before the first selection); either may be NULL. */
ESVO_API int esvo_hotpix_read(esvo_ctx* ctx, int cam, uint32_t* counts_or_null, uint8_t* mask_or_null);

/* Zeroes camera cam's counts and removes its mask: packed pushes are no longer filtered. */
ESVO_API int esvo_hotpix_clear(esvo_ctx* ctx, int cam);

/* *total = the number of events in camera cam's log since esvo_create / esvo_ts_reset: the `total` of the event windows
 * (esvo_events_window_dev, esvo_events_lower_bound_dev).  With a mask installed it counts the events the pushes kept.
 * Host-side state, no synchronisation. */
ESVO_API int esvo_ts_events_pushed(esvo_ctx* ctx, int cam, int64_t* total);

#ifdef __cplusplus
}
#endif
#endif /* ESVO_B200_HOTPIX_H_ */
