/*
 * esvo_b200_bag.h -- C ABI of the packed event ingest: dvs_msgs/EventArray events pushed to a camera's time surface as
 * they lie in a recorded ROS bag (include/esvo_b200/rosbag_events.hpp reads the bag).  esvo_b200.h includes this header.
 *
 * Kept apart from esvo_b200.h because the CPU oracle exports every declaration of esvo_b200.h under its own prefix; these
 * two have no oracle counterpart.  Their reference is esvo_ts_push_events on the decoded events: after the decode the two
 * paths are the same, and tests/test_gpu_bag_ingest.py holds them byte-identical.
 */
#ifndef ESVO_B200_BAG_H_
#define ESVO_B200_BAG_H_

#include "esvo_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces: TimeSurface::eventsCallback (TimeSurface.cpp:403-425) on a dvs_msgs/EventArray as it lies in a ROS bag.
 * The events are dvs_msgs/Event wire records: 13 bytes each, little-endian, no alignment:
 *   u16 x | u16 y | u32 sec | u32 nsec | u8 polarity
 * with stamp sec * 1e9 + nsec (ros::Time::toNSec) and polarity = (byte != 0).  The records are copied as they are and decoded
 * on the device.  Everything after the decode is esvo_ts_push_events on the decoded events: push indices, order check,
 * unordered mode, the fold of the resident log, error codes and messages.
 * runs[k] holds n_events[k] records (e.g. the event blocks of several EventArray messages of a memory-mapped bag); the
 * runs are gathered with memcpy into a pinned staging block of camera cam, then copied to the device in one transfer.
 * The runs may be reused as soon as the call returns; the work is enqueued and not waited for. */
ESVO_API int esvo_ts_push_event_array(esvo_ctx* ctx, int cam, const uint8_t* const* runs, const size_t* n_events,
                                      int n_runs);

/* esvo_ts_push_event_array on n wire records already in device memory at packed_dev (any byte alignment); enqueued on the
 * camera's stream, nothing is synchronised. */
ESVO_API int esvo_ts_push_event_array_dev(esvo_ctx* ctx, int cam, const uint8_t* packed_dev, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* ESVO_B200_BAG_H_ */
