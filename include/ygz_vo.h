/*
 * ygz_vo.h -- streaming C API of libygz_vo.so: the device-resident tracking engine (host/vo_driver.cpp) fed frame by
 * frame.  The reference's VisualOdometry::AddFrame (src/Module/VisualOdometry.cpp:38-107) takes one frame at a time; this
 * API takes frames as they arrive, per stream, and runs them in the engine's rounds: per stream a window of queued frames
 * up to the first one that may become a key-frame is tracked as one chain on the device, key-frames are inserted (Detect,
 * depth-initialised map points, local BA) behind it, and the BA overlaps the next round's alignment.  The results are
 * those of the batch entry points (ygz_vo_run_ex) on the same frames, whatever the pacing of push and step.
 *
 * Conventions are those of ygz_b200.h: YGZB_OK or a negative YGZB_ERR_* code, no exceptions, poses T_cw 3x4 row-major.
 *
 * Buffer lifetime: ygz_vo_push keeps the caller's pointers; no host copy is made.  An image and a depth map must stay
 * valid and unchanged until ygz_vo_poll has returned the result of that frame (the reference's Frame owns its _color and
 * _depth the same way).  Page-locked buffers (ygzb_host_alloc) make the uploads asynchronous.
 *
 * Depth: a frame's depth map (image_width * image_height doubles, metres, host or device memory) initialises the map
 * points of the key-frame the frame becomes; it is uploaded (ygzb_tracker_set_depth) only then, right before the
 * key-frame insertion.  NULL means the stream's current depth map stays valid: that of the last key-frame that had one.
 * A stream's first frame always becomes a key-frame, so it must have a depth map.
 *
 * Results: come out in frame order within each stream, each frame exactly once, and only when final.  A key-frame's pose
 * is its pose after its local BA, the value ygz_vo_run writes to its trajectory.  Once a stream is lost (its alignment
 * moved too far, or pose-only kept fewer than min_inliers inliers), that frame and every later one report
 * YGZ_VO_LOST with the last pose, until ygz_vo_restart starts a new sequence.  `frame` counts the stream's pushes from
 * 0, across restarts.
 *
 * Sequences: a stream's first frame becomes its first key-frame at the identity pose, or at the pose ygz_vo_restart set
 * before that push.  ygz_vo_restart on a stream that has frames starts a new sequence at the next push: nothing is
 * matched against the old one and none of its map is reused; the stream is bootstrapped exactly as a fresh one.
 *
 * Threading: one ygz_vo per context and host thread; the context's stream carries all of its work.
 */
#ifndef YGZ_VO_H_
#define YGZ_VO_H_

#include <stddef.h>
#include <stdint.h>

#include "ygz_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ygz_vo ygz_vo;

typedef struct {
    int n_streams;          /* independent sequences, >= 1                                                          */
    int window;             /* frames of one stream tracked per round at most, >= 1 (a result never depends on it)   */
    int ref_mode;           /* YGZB_TRACK_REF_KEYFRAME or YGZB_TRACK_REF_PREVIOUS (ygzb_tracker_set_reference_mode)  */
    int kf_min_frames;      /* NeedNewKeyFrame (VisualOdometry.cpp:304-321): frames since the last key-frame ...       */
    double kf_min_rot, kf_min_trans;   /* ... and the rotation (rad) or translation (m) from it that make a key-frame */
    int min_inliers;        /* pose-only inliers below which a stream is lost (vo.keyframe.min_features, 30)         */
    double K[4];            /* fx, fy, cx, cy in double; must round to the context's float fx..cy; the camera of
                               every stream until ygz_vo_set_camera gives it another                                 */
} ygz_vo_config;

#define YGZ_VO_TRACKED 0
#define YGZ_VO_KEYFRAME 1
#define YGZ_VO_LOST 2
typedef struct {
    int32_t stream, frame;
    int64_t tag;            /* the caller's tag of the frame (ygz_vo_push)                                          */
    int32_t status;         /* YGZ_VO_TRACKED, YGZ_VO_KEYFRAME or YGZ_VO_LOST                                       */
    int32_t n_inliers;      /* pose-only inliers (0 for a stream's first frame)                                     */
    double T_cw[12];
} ygz_vo_result;

/* A tracker on `ctx` for cfg->n_streams streams; the image size is the context's (ygzb_params image_width/height).
 * YGZB_ERR_INVALID for a NULL argument or a config that does not match the context.                                 */
int ygz_vo_create(ygzb_ctx* ctx, const ygz_vo_config* cfg, ygz_vo** out);
/* queues an image of `stream` (host or device memory) in the format of its sequence (ygz_vo_set_frame_format; by default
 * grey, image_width * image_height bytes): width * height * channels bytes, rows packed.  It is the raw, distorted frame
 * when the stream's sequence has a lens (ygz_vo_set_lens), which the engine resamples on the device as it uploads it; a
 * BGR frame is converted there.  Nothing runs until ygz_vo_step or ygz_vo_flush.  YGZB_ERR_INVALID, with nothing queued,
 * for a stream out of range, a NULL image, a NULL depth on a stream that has no depth map yet or whose next frame starts
 * a new sequence (ygz_vo_restart), or a sequence's first frame whose format has another size than the context's while the
 * sequence has no lens.                                                                                              */
int ygz_vo_push(ygz_vo* vo, int stream, const uint8_t* image, const double* depth, int64_t tag);
/* starts a new sequence of `stream` whose first key-frame takes pose T_cw (3x4 row-major; NULL: identity), to place a
 * sequence in the caller's world frame or to resume a lost stream, e.g. at the pose of its last YGZ_VO_LOST result.
 *  - Barrier: the frames pushed before the call belong to the old sequence and get exactly the results they would get
 *    without it -- tracked, key-frames (a pending key-frame insertion completes and its result comes first) or
 *    YGZ_VO_LOST.  No round tracks frames of both sequences together.
 *  - The first frame pushed after the call becomes the stream's first key-frame at T_cw; that push must bring a depth
 *    map.  From then on the stream is a fresh one: empty local map, key-frame ring and slots reused from the start, map
 *    point ids from 0, frames since the last key-frame, the lost flag and the previous-frame reference reset.  Its
 *    results are those of a fresh engine fed the same frames; ygz_vo_export_map holds only the new key-frames.
 *  - Before the stream's first push the call only sets the pose its first key-frame takes.  Of two calls with no push
 *    in between, the last one counts.
 *  - ygz_vo_stream_stats: counter 0 (lost) describes the current sequence, counter 12 counts the restarts that have
 *    started a sequence, the other counters keep accumulating.
 * The engine never restarts a stream by itself.  YGZB_ERR_INVALID, changing nothing, for a NULL vo, a stream out of
 * range, a non-finite entry, or a rotation that is not orthonormal with determinant +1 (within 1e-6 per entry).      */
int ygz_vo_restart(ygz_vo* vo, int stream, const double T_cw[12]);
/* K = {fx, fy, cx, cy} of `stream`'s next sequence, so that the streams of one engine may come from different cameras
 * (with the context's image size): the camera of the undistorted frames -- the frames as pushed, or with a lens
 * (ygz_vo_set_lens) the remapped ones, whose newK it is.  A camera belongs to a sequence:
 *  - Accepted before the stream's first push, or while a restart is pending (ygz_vo_restart called, nothing pushed
 *    since).  Of two calls with no push in between, the last one counts.
 *  - Barrier: frames pushed before ygz_vo_restart are tracked with the old camera, whatever is set afterwards; the new
 *    camera applies from the new sequence's first key-frame.
 *  - A stream with camera K gives the results, observation rows (in its own pixel frame), information records and map
 *    updates of a one-stream engine created with K on a context whose float fx..cy are (float)K.  K need not round to
 *    the context's camera.
 *  - ygz_vo_export_map carries the camera of the key-frames it holds (that of the stream's current sequence).  Stream
 *    records carry the stream's camera (the one its next push uses) in their header K, and ygz_vo_load_stream accepts a
 *    record only if that K equals the destination stream's camera bit for bit: to hand a stream with another camera
 *    over into a stream that has tracked, call ygz_vo_flush, ygz_vo_restart(stream) (a restart is then pending),
 *    ygz_vo_set_camera, then ygz_vo_load_stream.  The load replaces the whole state, the pending restart included; if it
 *    fails, the stream keeps the camera that was set and the restart stays pending.  A stream saved while a restart is
 *    pending after ygz_vo_set_camera carries the new camera, while its ring still holds the old sequence's key-frames;
 *    the loaded stream's ygz_vo_export_map reports them with the new camera until its next push restarts it (they are
 *    never tracked again).
 * YGZB_ERR_INVALID, changing nothing, for a NULL vo or K, a stream out of range, an entry that is not finite, fx <= 0 or
 * fy <= 0, or a call at any other time (the stream has pushed frames and no restart is pending).                 */
int ygz_vo_set_camera(ygz_vo* vo, int stream, const double K[4]);
/* the camera ygz_vo_set_camera last gave `stream` (the config's K until then): that of its current sequence, or of the
 * next one while a restart is pending.  YGZB_ERR_INVALID for a NULL vo or K or a stream out of range.               */
int ygz_vo_get_camera(const ygz_vo* vo, int stream, double K[4]);
/* the lens of `stream`'s next sequence, so that each stream may push raw frames of its own lens: K = {fx, fy, cx, cy} of
 * the raw camera and dist = {k1, k2, p1, p2, k3} (the model of ygzb_undistort_map); K = dist = NULL: no lens.
 *  - The sequence's frames are undistorted on the device as they are uploaded, level 0 being
 *    cv::remap(image, ygzb_undistort_map(width, height, K, dist, newK)) bit for bit, with newK the stream's camera for
 *    that sequence (ygz_vo_set_camera, or the config's K), and `image` the pushed frame, converted to grey first if it is
 *    BGR.  The raw frame may have its own size (ygz_vo_set_frame_format): K is then that raw camera's, the maps keep the
 *    context's width x height and taps outside the raw frame read 0.  With dist = 0 that is a pure crop or scale.  Everything else is in that undistorted camera: the depth maps
 *    pushed with the frames, the results, observation rows, information records, map updates and ygz_vo_export_map;
 *    the key-frame images of map and reference records are undistorted level 0 and are never remapped again.
 *  - A stream with a lens gives what a stream without one gives when it is pushed the undistorted frames.  A stream
 *    without a lens uploads exactly as before: no remap kernel, no map copy.
 *  - Accepted at the times ygz_vo_set_camera is; of two calls with no push in between, the last one counts.  The two
 *    calls may come in either order: the maps are built from the camera the sequence ends up with, when its first frame
 *    is uploaded.
 *  - Barrier: frames pushed before ygz_vo_restart are remapped with the old lens (or none) even when they are uploaded
 *    after the call; the new maps reach the device behind the last of them, without waiting for a local BA in flight.
 *  - The tracker holds 6 bytes of maps per pixel for each stream that has had a lens (1.8 MB at 640x480).
 *  - Clearing the lens of a sequence whose frame format has another size than the context's makes its first push fail.
 *  - Stream records of a stream with a lens are version 2 (a lens block behind the header), and ygz_vo_load_stream
 *    accepts a record only if its lens, or the absence of one, equals the destination stream's bit for bit (as for K).
 *    To hand a stream over into a stream that has tracked: ygz_vo_flush, ygz_vo_restart(stream), ygz_vo_set_camera,
 *    ygz_vo_set_lens, then ygz_vo_load_stream.
 * YGZB_ERR_INVALID, changing nothing, for a NULL vo, only one of K and dist, an entry that is not finite, fx <= 0 or
 * fy <= 0, a stream out of range, or a call at any other time.                                                     */
int ygz_vo_set_lens(ygz_vo* vo, int stream, const double K[4], const double dist[5]);
/* the lens ygz_vo_set_lens last gave `stream`: that of its current sequence, or of the next one while a restart is
 * pending.  *has_lens = 0 (K and dist zeros) for none.  YGZB_ERR_INVALID for a NULL argument or a stream out of range. */
int ygz_vo_get_lens(const ygz_vo* vo, int stream, int* has_lens, double K[4], double dist[5]);
/* the format of the frames `stream`'s next sequence pushes, so that each stream may come from a sensor of its own size and
 * colour: width x height pixels of `channels` bytes, 1 (grey) or 3 (BGR, converted as cv::cvtColor(COLOR_BGR2GRAY)), rows
 * packed.  The default, image_width x image_height x 1, is the frames as they have always been pushed.
 *  - A width x height other than the context's needs a lens (ygz_vo_set_lens) whose K is the raw camera's: level 0 is
 *    cv::remap(cvtColor(raw), ygzb_undistort_map(image_width, image_height, K, dist, newK)) bit for bit, newK the stream's
 *    camera.  The resampling is INTER_LINEAR, so a downscale of 2x or more aliases, exactly as cv::remap does.
 *  - Everything downstream keeps the context's size and the stream's camera: pyramid, grid, the depth maps pushed with
 *    the frames (image_width x image_height doubles), results, observation rows, information records, map updates and
 *    ygz_vo_export_map.  A stream with a format gives, byte for byte, what a default-format stream gives when it is
 *    pushed the frames resampled beforehand.  A stream of the default format without a lens uploads exactly as before.
 *  - Accepted at the times ygz_vo_set_camera is; of two calls with no push in between, the last one counts.
 *  - Barrier: frames pushed before ygz_vo_restart are uploaded with the old format even when they are uploaded after the
 *    call.
 *  - Stream records of a stream with a format other than the default are version 3 (a format block behind the header),
 *    and ygz_vo_load_stream accepts a record only if its format equals the destination stream's.
 * YGZB_ERR_INVALID, changing nothing, for a NULL vo, a stream out of range, a width or height < 1 or > 32767, channels
 * other than 1 and 3, or a call at any other time.                                                                 */
int ygz_vo_set_frame_format(ygz_vo* vo, int stream, int width, int height, int channels);
/* the format ygz_vo_set_frame_format last gave `stream` (the default until then): that of its current sequence, or of
 * the next one while a restart is pending.  YGZB_ERR_INVALID for a NULL argument or a stream out of range.           */
int ygz_vo_get_frame_format(const ygz_vo* vo, int stream, int* width, int* height, int* channels);
/* one round over what is queued, with one host synchronisation: the results of the windows it tracks are final on
 * return, except a frame that triggers a key-frame, whose insertion is enqueued by the next round.                 */
int ygz_vo_step(ygz_vo* vo);
/* rounds until nothing is queued or in flight: every pushed frame has its result                                    */
int ygz_vo_flush(ygz_vo* vo);
/* moves up to `capacity` final results, oldest first, into `out`; *n = how many.  With observations or information on,
 * the rows and records of the results it returns are discarded.                                                    */
int ygz_vo_poll(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n);

/* ---- observations: the map points each result's pose rests on (ygzb_observation, ygz_b200.h) --------------------------
 * on != 0: every result final from here on carries its frame's pose-only inliers as observation rows (map point id,
 * measured pixel, world point), in candidate order.  A result brings exactly n_inliers rows: a tracked frame's, a
 * key-frame's (the rows its map record's obs_id / obs_px hold), a YGZ_VO_LOST frame whose pose-only kept too few
 * inliers (its pose is the last good one); a sequence's first key-frame and a LOST frame after that bring none.  The
 * tracker writes them into a page-locked buffer of n_streams * window * YGZB_TRACK_RING * cells rows (48 bytes each:
 * 37.7 MB at 8 streams, window 8 and 3,072 cells), allocated when switched on and freed when switched off.  Stream
 * records do not carry observations.  YGZB_ERR_INVALID, changing nothing, unless the engine is idle: nothing queued,
 * no key-frame insertion pending, no result waiting to be polled.                                                  */
int ygz_vo_set_observations(ygz_vo* vo, int on);
/* ygz_vo_poll with the rows: moves whole results, oldest first, while they fit in `capacity` results and
 * `obs_capacity` rows; result k's out[k].n_inliers rows follow those of result k - 1 in `obs`; *n results, *n_obs rows.
 * YGZB_ERR_CAPACITY, moving nothing (*n = 0), when the rows of the first waiting result do not fit: *n_obs = its row
 * count.  YGZB_ERR_INVALID for a NULL vo, n or n_obs, a NULL out or obs with a capacity, or observations off.       */
int ygz_vo_poll_observations(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n, ygzb_observation* obs, size_t obs_capacity,
                             size_t* n_obs);

/* ---- pose information: how well each result's pose is determined (ygzb_pose_information, ygz_b200.h) -----------------
 * on != 0: every result final from here on carries an information record: the sparse alignment's Fisher information
 * (SparseImgAlign::getFisherInformation) and pose-only's information matrix of the returned T_cw, both as packed upper
 * triangles of symmetric 6x6 matrices.  Which record a result carries:
 *   YGZ_VO_TRACKED    its tracking job's;
 *   YGZ_VO_KEYFRAME   its tracking job's, computed at the tracked pose BEFORE the key-frame's local BA (the result's
 *                     T_cw is the pose after it);
 *   a sequence's first key-frame and every YGZ_VO_LOST result: all zeros.
 * The records do not depend on the window or the pacing.  The tracker writes them into a page-locked buffer of
 * n_streams * window records (336 bytes each), allocated when switched on and freed when switched off.  Stream records
 * do not carry them.  YGZB_ERR_INVALID, changing nothing, unless the engine is idle (as ygz_vo_set_observations).     */
int ygz_vo_set_information(ygz_vo* vo, int on);
/* one poll for both attachments: moves whole results, oldest first, into `out`; info[k] is out[k]'s record.  info must
 * be non-NULL exactly when information is on (room for `capacity` records).  With observations on, obs, obs_capacity and
 * n_obs follow ygz_vo_poll_observations (YGZB_ERR_CAPACITY included); with observations off obs must be NULL and
 * obs_capacity 0, and n_obs (may be NULL) is set to 0.  YGZB_ERR_INVALID for a NULL vo or n, a NULL out with a capacity,
 * or attachments that do not match what is switched on.                                                            */
int ygz_vo_poll_ex(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n, ygzb_pose_information* info, ygzb_observation* obs,
                   size_t obs_capacity, size_t* n_obs);

/* ---- map updates: the local map as each key-frame insertion leaves it (ygzb_map_point, ygz_b200.h) --------------------
 * A YGZ_VO_KEYFRAME result gives the key-frame's pose after its own local BA, but the BA also moves the older local
 * key-frames (all but the oldest, which fixes the gauge) and the points at least two local key-frames observe.  With map
 * updates on, every key-frame insertion brings one update: what it changed in the stream's local map.
 *   - n_local, local_frame, T_cw: the local key-frames after the insertion, oldest first, by frame index, and their poses
 *     as the ring holds them (the BA's, or the start pose for a sequence's first key-frame).  The last one is the new
 *     key-frame; its T_cw equals its YGZ_VO_KEYFRAME result's bit for bit.
 *   - n_moved rows: the BA's points in its landmark order (local key-frame, then feature); 0 for a first key-frame.
 *   - n_new rows: the new key-frame's points, ids mp0 .. mp0 + n_new - 1 in feature order.
 *   - retired_frame: the key-frame that left the local key-frames with this insertion, or -1.  No later BA includes it,
 *     so its pose and the points it created are final for the sequence.
 * Rows carry the positions the ring holds after the BA's write-back.  The two row sets never overlap, and a caller who
 * applies every update in order holds the engine's map -- every pose and point ygz_vo_export_map would give -- at any
 * time.  Map point ids restart from 0 with each sequence (ygz_vo_restart): key points by (stream, sequence, id).  A
 * restart retires nothing: the new sequence's first update has sequence + 1, n_local 1, and the old sequence's
 * key-frames are final as they were last reported.  The engine never revises a result: a caller who wants a tracked
 * frame to follow a later move of the key-frame it was tracked against (the newest key-frame before it) keeps the
 * relative pose, T_cw' = T_cw * T_kf^-1 * T_kf', with T_kf that key-frame's pose when the frame's result was final and
 * T_kf' its pose from a later update.  A lost stream inserts no key-frame, so it brings no update until it is restarted. */
typedef struct {
    int32_t stream;            /* the caller's stream index                                                        */
    int32_t frame;             /* the key-frame's frame index, the same as its YGZ_VO_KEYFRAME result's            */
    int64_t sequence;          /* restarts of the stream before this key-frame (ygz_vo_stream_stats counter 12)    */
    int32_t n_local;           /* local key-frames after the insertion (1 .. 3)                                    */
    int32_t retired_frame;     /* frame index of the key-frame that stopped being local, or -1                     */
    int32_t local_frame[YGZB_TRACK_RING];   /* their frame indices, oldest first; -1 past n_local                  */
    int32_t n_moved, n_new;    /* row counts: the BA's points, then the new key-frame's points                     */
    double T_cw[YGZB_TRACK_RING][12];       /* their poses (3x4 row-major) after the insertion; zeros past n_local */
} ygz_vo_map_update;           /* 432 bytes */
/* on != 0: every key-frame insertion final from here on queues its update, in a queue of its own (ygz_vo_poll and
 * ygz_vo_poll_ex neither return nor discard updates).  An update is queued when its YGZ_VO_KEYFRAME result is.  The
 * tracker writes the rows into a page-locked buffer of n_streams * YGZB_TRACK_RING * cells rows (32 bytes each: 3.1 MB at
 * 8 streams and 3,072 cells), allocated when switched on and freed when switched off.  Stream records and the batch
 * entry points do not carry updates.  YGZB_ERR_INVALID, changing nothing, unless the engine is idle (as
 * ygz_vo_set_observations); with updates on, idle also means no update waiting to be polled, for this call,
 * ygz_vo_set_observations and ygz_vo_set_information alike.                                                          */
int ygz_vo_set_map_updates(ygz_vo* vo, int on);
/* moves whole updates, oldest first, while they fit in `capacity` updates and `row_capacity` rows; update k's
 * out[k].n_moved + out[k].n_new rows follow those of update k - 1 in `rows`; *n updates, *n_rows rows.
 * YGZB_ERR_CAPACITY, moving nothing (*n = 0), when the rows of the first waiting update do not fit: *n_rows = its row
 * count.  YGZB_ERR_INVALID for a NULL vo, n or n_rows, a NULL out or rows with a capacity, or map updates off.     */
int ygz_vo_poll_map_updates(ygz_vo* vo, ygz_vo_map_update* out, int capacity, int* n, ygzb_map_point* rows, size_t row_capacity,
                            size_t* n_rows);
/* the 16 counters ygz_vo_run reports per stream: lost, key-frames, local BAs, candidates, projected, inliers, BA
 * observations, BA points, BA key-frames, BA LM trials, BA iterations, BA model FLOP, restarts (ygz_vo_restart),
 * 0, 0, 0                                                                                                         */
int ygz_vo_stream_stats(ygz_vo* vo, int stream, int64_t stats[16]);
/* the local map of `stream` (every key-frame still in its ring, oldest first) into `out`, sized for YGZB_TRACK_RING
 * key-frames (ygzb_tracker_export), with the stream's camera in out->K (ygz_vo_set_camera): asynchronous, valid after
 * ygzb_synchronize(ctx); call after ygz_vo_flush                                                                   */
int ygz_vo_export_map(ygz_vo* vo, int stream, ygzb_map_record* out);

/* ---- stream records: a live stream as plain bytes, to move it to another engine, context, device or process ----------
 * A stream record is the whole state of one stream: its host bookkeeping, its local map (ygzb_tracker_export), in
 * previous-frame mode its reference (ygzb_tracker_export_reference) and the depth map its next key-frame pushed with
 * depth = NULL would use (ygzb_tracker_get_depth).  A stream loaded from it continues exactly as the saved one would have.
 *
 * Layout: little-endian, packed (no padding; fields are not aligned), every count before the rows it describes.
 *   1. header      u8 magic[4] = "YGZS", u32 version = 1 (no lens, default format), 2 (a lens, default format) or 3
 *                  (a format other than the default), u64 size (of the whole record),
 *                  i32 width, height, cells, n_levels, f64 K[4] (the stream's camera), i32 ref_mode           (68 bytes)
 *      format      (version 3 only) i32 width, height, channels: the stream's frame format
 *                  (ygz_vo_get_frame_format), i32 has_lens (0 or 1)                                             (16 bytes)
 *      lens        (version 2, and version 3 with has_lens) f64 K[4], f64 dist[5]: the stream's lens
 *                  (ygz_vo_get_lens)                                                                            (72 bytes)
 *   2. host state  i32 n_kf, then per key-frame of the stream's ring, oldest first:
 *                      i32 entry, i32 n, i32 frame_id, i64 mp0, f64 T_cw[12]                               (116 bytes)
 *                  f64 T_cw[12] (current pose), f64 start[12] (pose of the next sequence's first key-frame),
 *                  u8 restart_pending, has_pose, lost, has_depth (0 or 1),
 *                  i32 frames_since_kf, i32 next_frame (the frame index of the stream's next push), i64 next_mp,
 *                  i64 counters[11] (stats 1-10 and 12 of ygz_vo_stream_stats), f64 ba_flops
 *   3. map         i32 n_keyframes (= n_kf), then per key-frame:
 *                      i32 entry, i32 n_features, i32 n_obs, i64 mp0, f64 T_cw[12], u8 image[height][width]
 *                  then the live rows of all key-frames, key-frame after key-frame (F = sum n_features, O = sum n_obs):
 *                      f64 px[F][2], u8 level[F], f64 depth[F], f64 pw[F][3], i64 obs_id[O], f64 obs_px[O][2]
 *   4. reference   (ref_mode YGZB_TRACK_REF_PREVIOUS and n_kf > 0 only)
 *                  i32 n, f64 T_cw[12], f64 px[n][2], f64 depth[n], u8 image[height][width]
 *   5. depth       (has_depth only) f64 depth[height][width]
 * The fields are those of ygzb_map_record and ygzb_reference_record; a stream never pushed is a record of sections 1-2
 * and an empty map.                                                                                                 */
#define YGZ_VO_STREAM_RECORD_VERSION 1
#define YGZ_VO_STREAM_RECORD_VERSION_LENS 2
#define YGZ_VO_STREAM_RECORD_VERSION_FORMAT 3
/* *bytes = an upper bound of the size of any stream record of `vo`: a full ring, a full reference, a depth map, while a
 * stream of `vo` has a lens (ygz_vo_get_lens) the lens block, and while one has a format other than the default
 * (ygz_vo_get_frame_format) the format block.                                                                         */
int ygz_vo_stream_record_bound(const ygz_vo* vo, size_t* bytes);
/* the whole state of `stream` as a record in buf[0 .. *size).  Synchronous: it synchronises the context.
 *  - The stream must have no queued frame and no pending key-frame insertion (ygz_vo_flush first), so that every frame
 *    pushed to it has its final result; other streams of `vo` may have queued frames, which stay queued.
 *  - It does not change the stream: the saved stream may go on tracking, and the record then forks it.
 * YGZB_ERR_INVALID, changing nothing, for a NULL vo or size, a NULL buf with capacity > 0, a stream out of range, or a
 * stream with queued frames or a pending insertion; YGZB_ERR_CAPACITY if the record does not fit in `capacity` bytes
 * (*size = its size; buf = NULL, capacity = 0 asks for the size).                                                   */
int ygz_vo_save_stream(ygz_vo* vo, int stream, void* buf, size_t capacity, size_t* size);
/* `stream` of vo continues the saved stream: its whole state, counters included, is replaced by the record's, and its
 * next push is the saved stream's next frame (frame index and results as the saved stream would have given them).
 *  - The destination stream must have no queued frame and no pending key-frame insertion; results already waiting in
 *    the result queue stay there for ygz_vo_poll.
 *  - The engine may differ from the saved one in n_streams, window, key-frame policy and min_inliers (the destination's
 *    apply from here on), in the stream index and in its context and device.  It must match it in image size, grid
 *    cells, pyramid levels and ref_mode, and the destination stream's camera (ygz_vo_get_camera) must equal the
 *    record's K bit for bit, its lens (ygz_vo_get_lens) the record's lens, or have none for a version-1 record, and its
 *    frame format (ygz_vo_get_frame_format) the record's, or be the default for a version-1 or -2 record.
 *  - The record is checked whole on the host before anything is enqueued.
 * Asynchronous like ygzb_tracker_import; `buf` may be released when the call returns.  YGZB_ERR_INVALID, with the
 * stream exactly as before, for a NULL vo or buf, a stream out of range or with queued frames or a pending insertion,
 * a wrong magic or version, a size that is not the record's, a different geometry, K, lens, format or ref_mode, a count, entry,
 * level or pose out of range, or a host state no saved stream can have (e.g. frames pushed but no key-frame, key-frames
 * but no frame pushed, map sections that disagree with the host state).                                            */
int ygz_vo_load_stream(ygz_vo* vo, int stream, const void* buf, size_t size);

void ygz_vo_destroy(ygz_vo* vo);

#ifdef __cplusplus
}
#endif

#endif /* YGZ_VO_H_ */
