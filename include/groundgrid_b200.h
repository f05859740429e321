/*
 * groundgrid_b200 -- C-ABI of the H100-native GroundGrid per-scan hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  The host
 * classes in groundgrid_b200/host (groundgrid::GroundGrid / groundgrid::GroundSegmentation,
 * same surface as the reference headers) are thin wrappers over these calls; a maintainer
 * of the reference binds them exactly the same way (see INTEGRATION.md).
 *
 * Every entry point cites the reference interface it replaces (paths relative to the
 * dcmlr/groundgrid repository).  All functions return 0 on success or a negative GG_E_* code;
 * no exception crosses this boundary.  A handle is not thread-safe (same contract as the
 * reference: callbacks are serialised on one ROS queue, src/GroundGridNodelet.cpp:79).
 *
 * There is NO CPU fallback: every compute entry point fails with GG_E_CUDA when no sm_90
 * device is usable.
 *
 * Data layout at the boundary (SURVEY.md section 8b):
 *   - points: 32-byte PointXYZIR records (include/velodyne_pointcloud/point_types.h:27-33)
 *   - layers: N x N float, column-major like Eigen::MatrixXf: element (i, j) at i + j*N,
 *     row index i grows toward -x, column index j toward -y (grid_map convention).
 *   - one handle owns `n_slots` independent maps ("slots"); slot s is what one
 *     GroundGrid + GroundSegmentation pair owns in the reference: its map and its
 *     configuration (gg_set_slot_config).  n_slots == 1 is the plain drop-in; n_slots > 1 is
 *     the batched throughput mode (independent scans, e.g. of sensors with different
 *     settings, in one launch).
 */
#ifndef GROUNDGRID_B200_H
#define GROUNDGRID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GG_OK 0
#define GG_E_ARG (-1)      /* bad argument (null pointer, slot out of range, too many points ...) */
#define GG_E_CUDA (-2)     /* CUDA runtime error or no usable device; see gg_last_error() */
#define GG_E_STATE (-3)    /* map not initialised (reference: points_callback returns early, GroundGridNodelet.cpp:124-125) */
#define GG_E_LAYER (-4)    /* unknown layer name (reference: std::out_of_range from grid_map) */

#define GG_LABEL_ABSENT 0      /* point is not part of the output cloud (outside map / NaN / border cell) */
#define GG_LABEL_GROUND 49     /* src/GroundSegmentation.cpp:180,188 */
#define GG_LABEL_NONGROUND 99  /* src/GroundSegmentation.cpp:175 */

/* gg_create flags */
#define GG_FLAG_FULL_LAYERS 1u /* also maintain the layers the algorithm never reads back
                                  (groundCandidates, planeDist, m2, meanVariance, pointsRaw,
                                  maxGroundHeight; src/GroundSegmentation.cpp:61-67,234,296,303,307) */

/* include/velodyne_pointcloud/point_types.h:27-33 -- velodyne_pointcloud::PointXYZIR, sizeof == 32 */
typedef struct gg_point {
    float x, y, z, _pad0;
    float intensity;
    uint16_t ring;
    uint16_t _pad1;
    float _pad2[2];
} gg_point;

/* cfg/GroundGrid.cfg:8-21 -- groundgrid::GroundGridConfig (same order, same defaults) */
typedef struct gg_config {
    int point_count_cell_variance_threshold;                     /* 10 */
    int max_ring;                                                /* 1024 */
    double groundpatch_detection_minimum_threshold;              /* 0.01 (declared, never read) */
    double distance_factor;                                      /* 0.0001 */
    double minimum_distance_factor;                              /* 0.0005 */
    double miminum_point_height_threshold;                       /* 0.3 */
    double minimum_point_height_obstacle_threshold;              /* 0.1 */
    double outlier_tolerance;                                    /* 0.1 */
    double ground_patch_detection_minimum_point_count_threshold; /* 0.25 */
    double patch_size_change_distance;                           /* 20 */
    double occupied_cells_decrease_factor;                       /* 5 */
    double occupied_cells_point_count_factor;                    /* 20 */
    double min_outlier_detection_ground_confidence;              /* 1.25 */
    int thread_count;                                            /* 8 (accepted, unused: no host threads) */
} gg_config;

typedef struct gg_handle_s* gg_handle;

/* Per-scan inputs of one slot (arguments of GroundSegmentation::filter_cloud,
 * include/groundgrid/GroundSegmentation.h:55):
 *   origin  = cloudOrigin (x, y, z of the sensor in the map frame, GroundGridNodelet.cpp:139-146,190-194)
 *   base_z  = z of mapToBase * (0,0,0) (GroundSegmentation.cpp:405-411)
 *   flags   = GG_SCAN_DEVICE_POSE: origin / base_z come from the slot's device scan pose (gg_update_poses_from_device)
 *             instead of this descriptor; the other bits are reserved and ignored (pass 0)                */
#define GG_SCAN_DEVICE_POSE 1
typedef struct gg_scan_desc {
    int slot;
    int flags;
    size_t n_points;
    float origin[3];
    float _pad;
    double base_z;
} gg_scan_desc;

/* Fills *cfg with the defaults of cfg/GroundGrid.cfg:8-21. */
void gg_default_config(gg_config* cfg);

/* Text of the last error on this thread (CUDA error string or argument complaint). */
const char* gg_last_error(void);

/* Replaces GroundSegmentation::init (src/GroundSegmentation.cpp:37-48: builds the expectedPoints
 * table for round(dimension/resolution)^2 cells) plus the device-side allocation of `n_slots`
 * maps.  `max_points` is the per-scan capacity.  `stream` is a cudaStream_t (NULL = the handle
 * creates its own non-blocking streams).  `device` is the CUDA ordinal. */
int gg_create(double dimension_m, float resolution, int device, int n_slots, size_t max_points,
              unsigned flags, void* stream, gg_handle* out);
int gg_destroy(gg_handle h);

int gg_cells_per_side(gg_handle h);  /* N (364 for the reference default 120 m / 0.33 m) */
int gg_num_slots(gg_handle h);

/* Replaces GroundGrid::setConfig + GroundSegmentation::setConfig
 * (src/GroundGrid.cpp:48, src/GroundSegmentation.cpp:468-471; GroundGridNodelet.cpp:299-302). */
int gg_set_config(gg_handle h, const gg_config* cfg);
int gg_get_config(gg_handle h, gg_config* cfg);
/* gg_set_config is handle-wide: it waits for all work of the handle, then sets every slot's configuration
 * (replacing per-slot settings); gg_get_config returns what it last set (the defaults until then). */

/* GroundSegmentation::setConfig / GroundGrid::setConfig of the pair that owns slot `slot`
 * (src/GroundSegmentation.cpp:468-471, src/GroundGrid.cpp:48, GroundGridNodelet.cpp:299-302).
 * A slot starts with the handle-wide configuration and keeps its own through gg_init_map, rolls and
 * configuration changes of other slots.  The new configuration applies from the slot's next launch on
 * (every path: gg_filter_cloud[_batch[_begin]], gg_run_scans[_device], the per-phase entries).
 * gg_set_slot_config waits only for the work already enqueued on the slot's stream group; other groups keep
 * running with their own configurations.  (That stream may itself wait on work of other groups -- after
 * gg_fork_streams / gg_join_streams -- and such work is then waited for as well.)  A
 * gg_filter_cloud_batch_begin batch that contains the slot must be waited for (gg_filter_cloud_batch_wait or
 * gg_synchronize) first.  Slots with identical settings share one copy of the derived device data.  thread_count is accepted and unused.  GG_E_ARG: null handle or config,
 * slot out of range; values are not validated (like gg_set_config). */
int gg_set_slot_config(gg_handle h, int slot, const gg_config* cfg);
int gg_get_slot_config(gg_handle h, int slot, gg_config* cfg);

/* Replaces GroundGrid::initGroundGrid (src/GroundGrid.cpp:50-80): map centred on (x, y),
 * ground = z, groundpatch = 1e-7, points = 0, min = 100, max = -100. */
int gg_init_map(gg_handle h, int slot, double x, double y, double z);

/* Replaces GroundGrid::update for an already initialised map (src/GroundGrid.cpp:83-147):
 * rolls the map to the odometry position (x, y) by whole cells, seeds exposed cells with
 * ground = -(T * (cx, cy, 0)).z and groundpatch = 0 where T = row-major 3x4 [R|t] of
 * lookupTransform("base_link", "map").  *moved (may be NULL) = 1 if a cell shift happened. */
int gg_update_pose(gg_handle h, int slot, double x, double y, const double T_base_from_map[12], int* moved);

/* Batched gg_update_pose: `count` distinct slots (a repeated slot is GG_E_ARG), xy = 2 doubles per slot, T = 12 doubles per
 * slot, moved (may be NULL) = 1 int per slot.  One roll launch covers all slots. */
int gg_update_pose_batch(gg_handle h, int count, const int* slots, const double* xy, const double* T, int* moved);

/* Current map centre position (grid_map::GridMap::getPosition()).  On a slot whose position is device-owned (a
 * gg_update_poses_from_device roll since the host last knew it), gg_get_map_position, gg_update_pose[_batch],
 * gg_set_map_position and gg_init_map first WAIT on the host for the work enqueued on the slot's stream group, take
 * the position back (the slot is host-owned again) and then proceed as on a host-owned slot. */
int gg_get_map_position(gg_handle h, int slot, double xy[2]);

/* ---- poses from caller GPU memory ----
 * The per-step pose inputs of GroundGrid::update (src/GroundGrid.cpp:83-147: the odometry position and
 * lookupTransform("base_link", "map")) and of points_callback (src/GroundGridNodelet.cpp:127-146: cloudOrigin and the z
 * of mapToBase), for `count` distinct slots, read from DEVICE memory and resolved on the device, ordered on the
 * caller's stream.  For callers whose poses are produced on the GPU (GPU odometry or localization, simulators,
 * sequences replayed from HBM), which would otherwise copy them to the host every step.
 * Entry k of every array belongs to slots[k]; all pointers are DEVICE pointers on the handle's device. */
typedef struct gg_device_poses {
    const double* xy;               /* [count][2] or NULL: odometry position (GroundGrid::update, inOdom position), 8-byte aligned */
    const double* T_base_from_map;  /* [count][12] row-major 3x4 lookupTransform("base_link", "map"); NULL iff xy is */
    const float* origin;            /* [count][3] or NULL: cloudOrigin of the slot's next scans, 4-byte aligned */
    const double* base_z;           /* [count] or NULL: z of mapToBase * (0,0,0); NULL iff origin is */
} gg_device_poses;

/* Roll (xy given): per slot, bit-identical to gg_update_pose_batch with the same values at the same point of the slot's
 *   stream -- the new map position, the rolled "ground" / "groundpatch" and the seeded cells.  The cell shift is resolved
 *   on the device in fp64 exactly as the host does it.  dev_moved (int32 [count], 4-byte aligned, may be NULL):
 *   dev_moved[k] = 1 if the cells shifted, 0 if not, and -1 if xy[k] is not finite or the cell shift does not fit in
 *   int32; a -1 slot keeps its map and position untouched.  Afterwards the slot's position is device-owned: every later
 *   launch that needs it (scans, per-phase entries, gg_sample_layers_to_device, rolls) reads it from the device in
 *   stream order, and the host calls listed at gg_get_map_position wait for it.
 * Scan pose (origin given): stored per slot on the device.  Every later scan of the slot whose gg_scan_desc sets
 *   GG_SCAN_DEVICE_POSE uses the latest stored pose in the slot's stream order instead of its descriptor's origin /
 *   base_z, with (float)base_z applied as for a host value.  The flag is honoured by gg_run_scans, gg_run_scans_device,
 *   gg_run_scans_to_device, gg_run_cloud_msgs_to_device, gg_run_merged_cloud_msgs_to_device and
 *   gg_filter_cloud_batch[_begin].  A flagged scan of a slot that has no device scan pose since its gg_init_map is
 *   GG_E_STATE.
 * stream: cudaStream_t; NULL is the legacy default stream.  The contract of gg_get_layers_to_device: the work starts
 *   after everything already enqueued on `stream` and on the stream groups of the slots, work enqueued on `stream`
 *   afterwards sees dev_moved, and nothing waits on the host except the flow control of the parameter staging ring.
 *   The poses are consumed by the first kernel of each stream group, so a stream-ordered allocator may free or refill
 *   them on `stream` right after the call.
 * gg_point_info_to_device on a slot with a device roll since its last scan is GG_E_STATE (the host cannot know whether
 * that roll moved the cells).
 * count == 0, or all four pointers NULL, returns GG_OK and enqueues nothing.  Rejected with nothing enqueued:
 *   GG_E_ARG   null handle, slots or poses; count > n_slots; a slot out of range or repeated; xy without
 *              T_base_from_map or the reverse; origin without base_z or the reverse; a misaligned pointer (8 bytes for
 *              the doubles, 4 for origin and dev_moved); dev_moved overlapping the inputs or the handle's layers
 *   GG_E_STATE a slot whose map is not initialised
 * As for every call: a gg_filter_cloud_batch_begin batch that touches the same slots needs a gg_synchronize (or its
 * _wait) first. */
int gg_update_poses_from_device(gg_handle h, int count, const int* slots, const gg_device_poses* poses, int32_t* dev_moved,
                                void* stream);

/* Replaces GroundSegmentation::filter_cloud (src/GroundSegmentation.cpp:50-197) for one slot with
 * HOST buffers: copies the cloud to the device, runs rasterise -> patch detection -> spiral
 * interpolation -> labelling, copies results back and returns when they are in host memory.
 *   labels_out : n bytes, per INPUT point: 0 absent / 49 ground / 99 non-ground   (may be NULL)
 *   index_out  : n_out uint32, input index of each output point in the reference's output
 *                order: kept, then ignored, then outliers (:112-117,150,185)        (may be NULL)
 *   cloud_out  : n_out records, the reference's returned cloud (intensity = 49/99)  (may be NULL)
 *   n_out      : number of points in the output cloud                              (may be NULL) */
int gg_filter_cloud(gg_handle h, int slot, const gg_point* points, size_t n, const float origin[3],
                    double base_z, uint8_t* labels_out, uint32_t* index_out, gg_point* cloud_out,
                    size_t* n_out);

/* Batched form of gg_filter_cloud: `count` independent scans (distinct slots), host buffers.
 * points[k] / labels_out[k] are per-scan host pointers (pinned memory makes the copies
 * asynchronous).  Copies and kernels of different scans overlap on internal streams.
 * PCIe is the bottleneck of this path.  Host worker threads (GG_HOST_THREADS; default: the usable
 * CPUs of the process minus one) repack clouds into pinned staging memory as x | y | z | ring
 * (14 of the 32 bytes of a PointXYZIR record are used by the algorithm) so that only those bytes
 * cross the bus; whenever the packers fall behind the bus (fewer than two packed clouds queued for
 * copying), the calling thread sends scans from the back of the batch, which no packer has reached
 * yet, as plain 32-byte records.  GG_HOST_PACK=1 packs every scan, GG_HOST_PACK=0 none.  Results
 * are identical in all modes.  Every scan runs with its slot's configuration (gg_set_slot_config). */
int gg_filter_cloud_batch(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* points,
                          uint8_t* const* labels_out);

/* The same call in two halves, for callers that keep the bus busy across batches: _begin returns as
 * soon as every cloud has been handed to the copy engines and every kernel is enqueued; the labels of
 * that batch are complete after _wait(ticket) (or gg_synchronize).  At most two batches are in
 * flight: _begin first waits for the batch before the previous one.  points[k] and labels_out[k] of a
 * batch must stay untouched until its _wait; gg_update_pose_batch for the next scans may be called
 * right after _begin (stream order keeps roll -> scan -> roll -> scan per slot).  Other calls that
 * touch the same slots need a gg_synchronize first. */
int gg_filter_cloud_batch_begin(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* points,
                                uint8_t* const* labels_out, int* ticket);
int gg_filter_cloud_batch_wait(gg_handle h, int ticket);

/* Device-resident pipeline pieces (what gg_filter_cloud_batch is made of; used by bench.py to time
 * the kernels with the inputs already in HBM, and by the tests to check single phases):
 *   gg_upload_points : async H2D of one scan into its slot
 *   gg_run_scans     : enqueue the kernels for `count` scans whose points are resident.
 *                      stop_after: 0 whole path, 1 after rasterisation, 2 after patch detection,
 *                      3 after spiral interpolation
 *   gg_download_labels : async D2H of the per-input-point labels of one slot
 *   gg_synchronize   : wait for everything enqueued on the handle                              */
int gg_upload_points(gg_handle h, int slot, const gg_point* points, size_t n);
int gg_run_scans(gg_handle h, int count, const gg_scan_desc* scans, int stop_after);
int gg_download_labels(gg_handle h, int slot, uint8_t* labels_out, size_t n);
int gg_synchronize(gg_handle h);

/* The per-phase methods of the reference class, for callers that drive the phases themselves
 * (include/groundgrid/GroundSegmentation.h:56-62; all enqueue on the slot's stream):
 *   gg_run_scans(.., stop_after = 1)  = the layer reset of filter_cloud (:61-75) + insert_cloud over the whole cloud
 *                                       (:200-311); gg_get_point_classes then returns, per input point,
 *                                       class << 24 | cell with class 0 absent, 1 kept, 2 kept (border cell),
 *                                       3 ignored, 4 ignored (border cell), 5 outlier -- the contents of the
 *                                       point_index / ignored / outliers lists of :112-117
 *   gg_detect_ground_patches          = detect_ground_patches for all four sections (:314-340; sections are disjoint
 *                                       and every cell only writes itself, so their union is order-free).  Reads the
 *                                       planes "points" (whatever gg_get_layer's "points" names at the call: the kept-
 *                                       point count after a scan stopped before labelling, else the non-ground count),
 *                                       "minGroundHeight", "ground", "groundpatch", and writes "ground", "groundpatch".
 *                                       With GG_FLAG_FULL_LAYERS it first sets "variance" = m2 / (points + FLT_MIN)
 *                                       (:323) as the reference does; a handle without the flag keeps no "m2" and reads
 *                                       the stored "variance" in its place -- the one difference from the reference.
 *                                       Any float in these planes (NaN, +-inf, fractional or negative counts) gives the
 *                                       reference's result.
 *   gg_detect_ground_patch            = detect_ground_patch<patch_size>(map, i, j) for one cell (:343-395): reads
 *                                       "points" (as above), the stored "variance", "minGroundHeight", "ground",
 *                                       "groundpatch"; no variance recompute, as in the reference
 *   gg_spiral_ground_interpolation    = spiral_ground_interpolation (:398-441), base_z = z of toBase * (0,0,0)
 *   gg_interpolate_cell               = interpolate_cell(map, x, y) (:445-465)                                   */
int gg_get_point_classes(gg_handle h, int slot, uint32_t* codes, size_t n);
int gg_detect_ground_patches(gg_handle h, int slot);
int gg_detect_ground_patch(gg_handle h, int slot, int patch_size, int i, int j);
int gg_spiral_ground_interpolation(gg_handle h, int slot, double base_z);
int gg_interpolate_cell(gg_handle h, int slot, int x, int y);

/* Like gg_run_scans, but scan k reads its cloud from the caller-owned DEVICE buffer dev_points[k]
 * (n_points 32-byte records, 16-byte aligned) instead of the slot's upload buffer.  The buffer
 * must stay valid until the work is complete (and until gg_get_output, if that is used). */
int gg_run_scans_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* dev_points, int stop_after);

/* Caller-owned DEVICE destinations of one scan of gg_run_scans_to_device (on the handle's device; each may be NULL).
 * Each needs room for the scan's n_points entries. */
typedef struct gg_scan_outputs {
    uint8_t* labels;   /* per input point: 0 absent / 49 ground / 99 non-ground (the bytes gg_download_labels returns) */
    uint32_t* index;   /* input index of each selected output point, in the reference's output order (4-byte aligned) */
    gg_point* cloud;   /* the selected output points as records, intensity = 49 / 99, like gg_get_output (16-byte aligned) */
} gg_scan_outputs;

#define GG_SELECT_GROUND 1u     /* output points labelled 49 (outliers are always ground) */
#define GG_SELECT_NONGROUND 2u  /* output points labelled 99; both bits = the whole output cloud of filter_cloud */

/* gg_run_scans_device(.., stop_after = 0) with the results written into caller-owned device memory, ordered on the
 * caller's stream.  The slots' state afterwards is the same as after gg_run_scans_device (layers, gg_get_output,
 * gg_download_labels, gg_eval_accumulate), and so is the lifetime rule for dev_points.
 *   outs       : `count` entries (NULL: no outputs).  index / cloud of scan k receive the reference's output cloud
 *                (kept, then ignored, then outlier points, input order within each class) restricted to the labels in
 *                `select`: GG_SELECT_GROUND | GG_SELECT_NONGROUND gives exactly what gg_get_output gives,
 *                GG_SELECT_NONGROUND the obstacle cloud (kept and ignored points labelled 99, in that order).
 *   dev_counts : device int32[count]; dev_counts[k] = number of selected points of scan k, nothing is written past it.
 *                Required when any index or cloud is given; written whenever it is given and select != 0.
 *   stream     : cudaStream_t; NULL is the legacy default stream (not "unordered").  The call's device work starts
 *                after everything already enqueued on `stream`, and everything enqueued on `stream` after the call
 *                starts after all outputs are written (one event each way per stream group with scans in the batch).
 *                So with a stream-ordered allocator the caller may free the inputs or reuse the outputs' memory on
 *                `stream` right after the call.  The call does not wait on the host for device work, except for the
 *                flow control of the parameter staging ring (as every launching call).
 * GG_E_ARG, with nothing enqueued: what gg_run_scans_device rejects (GG_E_STATE for a map not initialised); index or
 * cloud with select 0; unknown select bits; index or cloud without dev_counts; index not 4-byte or cloud not 16-byte
 * aligned; an output range of a scan (its labels, index, cloud or dev_counts entry) that overlaps its own input cloud. */
int gg_run_scans_to_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* dev_points,
                           const gg_scan_outputs* outs, unsigned select, int32_t* dev_counts, void* stream);

/* ---- steps next to the path (SURVEY.md section 8f) -------------------------------------------
 * gg_upload_cloud_msg replaces pcl::fromROSMsg + the per-point tf2::doTransform loop of
 * GroundGridNodelet::points_callback (src/GroundGridNodelet.cpp:119-120,148-184): the raw
 * sensor_msgs/PointCloud2 payload (`point_step` bytes per point, fields x, y, z, intensity float32 and
 * ring uint16 at `field_offsets`, -1 = absent; e.g. {0,4,8,12,16} for the KITTI player's 18-byte points,
 * scripts/kitti_data_publisher.py:139-150) is copied to the device, unpacked into PointXYZIR records
 * and -- unless T is NULL (frame_id == "map") -- transformed with the row-major 3x4 T = lookupTransform
 * ("map", frame_id) in fp64.  The records land in the slot's cloud buffer: follow with gg_run_scans.
 *
 * gg_terrain_image replaces the "terrain" branch of publish_grid_map_layer (:247-270): N*N*3 floats,
 * pixel (i, j) = (ground, 3x3 pointsRaw sum >= 27 ? 1 : 0, pointsRaw); needs GG_FLAG_FULL_LAYERS.
 *
 * gg_eval_accumulate / gg_eval_read replace the tallies of scripts/eval_groundpoint_classifier.py:95-118:
 * counts[id][0] / counts[id][1] = points of ground-truth label `id` (taken from `ring`) predicted ground /
 * non-ground, accumulated over the scans it was called for (1024 ids). */
int gg_upload_cloud_msg(gg_handle h, int slot, const void* data, size_t n_points, int point_step, const int field_offsets[5],
                        const double T_map_from_frame[12]);

/* One sensor_msgs/PointCloud2 payload in DEVICE memory (on the handle's device).  The field rules are those of
 * gg_upload_cloud_msg: x, y, z, intensity float32 and ring uint16 at field_offsets, -1 = absent (x, y, z required). */
typedef struct gg_cloud_msg {
    const void* data;                /* n_points * point_step bytes, no alignment required */
    int point_step;
    int field_offsets[5];            /* x, y, z, intensity, ring */
    const double* T_map_from_frame;  /* HOST pointer, row-major 3x4 of lookupTransform("map", frame_id); NULL: frame_id == "map" */
} gg_cloud_msg;

/* The whole of GroundGridNodelet::points_callback after the lookups (src/GroundGridNodelet.cpp:119-120,148-184: pcl::fromROSMsg,
 * the per-point tf2::doTransform, filter_cloud) for a batch of payloads already in device memory.  For every scan k:
 *   1. msgs[k] (scans[k].n_points records) is unpacked into the slot's OWN cloud buffer and, when T_map_from_frame is
 *      given, transformed to the map frame in fp64 (the result per point is bit-identical to gg_upload_cloud_msg of the
 *      same bytes);
 *   2. then what gg_run_scans_to_device does follows on that buffer: outs, select, dev_counts and the stream contract
 *      are the same (NULL stream = the legacy default stream; the work starts after everything already enqueued on
 *      `stream`, work enqueued on `stream` afterwards sees the outputs complete; no host wait except the flow control of
 *      the parameter staging ring).
 * scans[k].origin is still the caller's (or, with GG_SCAN_DEVICE_POSE, the slot's device scan pose): the reference takes it
 * from a separate lookup, map <- velodyne (:131,139-146).
 * Consequences:
 *   - each payload is consumed by the first kernel of its slot's stream group, so a stream-ordered allocator may free
 *     it, or reuse its memory, on `stream` right after the call;
 *   - an output of scan k may overlap scan k's own payload (the output kernels read the slot's buffer, not the payload);
 *     buffers of different scans must not overlap;
 *   - T_map_from_frame is read during the call and may be reused when it returns;
 *   - the slots' state afterwards is what gg_upload_cloud_msg of the same bytes + gg_run_scans leaves: layers,
 *     gg_download_labels, gg_eval_accumulate, and gg_get_output without the payload having to stay alive.
 * count == 0 returns GG_OK and enqueues nothing.  GG_E_ARG, with nothing enqueued: what gg_run_scans_to_device rejects
 * except its input-overlap rule (GG_E_STATE for a map not initialised); null msgs; per message the layout rules of
 * gg_upload_cloud_msg: null data with n_points > 0, point_step < 12, x, y or z absent, a field outside point_step. */
int gg_run_cloud_msgs_to_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_cloud_msg* msgs,
                                const gg_scan_outputs* outs, unsigned select, int32_t* dev_counts, void* stream);

/* ---- a multi-LiDAR rig: several sensor payloads per scan ----
 * One scan of a rig with several sensors arrives as one PointCloud2 payload per sensor, each in its own frame.  The
 * reference sees such a rig as one cloud merged upstream in the map frame: every sensor's points go through
 * tf2::doTransform in fp64, are stored as float and are concatenated, and filter_cloud runs on the merged cloud with one
 * cloudOrigin.  These calls do that merge on the device, into the slot's own cloud buffer. */
#define GG_MAX_CLOUD_PARTS 16

/* One sensor's payload of a merged scan: the layout and frame rules of gg_cloud_msg, and its own point count.
 * msg.data is DEVICE memory for gg_run_merged_cloud_msgs_to_device and HOST memory for gg_upload_cloud_msgs;
 * msg.T_map_from_frame is a HOST pointer in both (NULL: the part is already in the map frame). */
typedef struct gg_cloud_part {
    gg_cloud_msg msg;
    size_t n_points;
} gg_cloud_part;

/* gg_run_cloud_msgs_to_device for scans made of several payloads.  Scan k owns the next n_parts[k] entries of `parts`,
 * taken in order (0 <= n_parts[k] <= GG_MAX_CLOUD_PARTS).  Part p of scan k is unpacked and, when it has a
 * T_map_from_frame, transformed into the slot's own cloud buffer from record sum(n_points of the scan's parts before p)
 * on; per point the result is bit-identical to gg_upload_cloud_msg of the same bytes.  scans[k].n_points must equal the
 * sum of its parts' n_points, and the scan then runs on the whole buffer exactly as in gg_run_cloud_msgs_to_device:
 * outs, select, dev_counts, the stream contract (the work, including every part's unpack, starts after everything
 * already enqueued on `stream`; no host wait except the flow control of the parameter staging ring), payloads that may
 * be freed on `stream` right after the call, outputs that may overlap their own scan's parts, and the slots' state
 * afterwards (layers, gg_get_output, gg_eval_counts_to_device / gg_eval_accumulate read the slot's buffer).
 * scans[k].origin is the single cloudOrigin of the merged scan.  A scan with no parts and n_points == 0 is empty.
 * count == 0 returns GG_OK and enqueues nothing.  GG_E_ARG, with nothing enqueued: what gg_run_cloud_msgs_to_device
 * rejects (GG_E_STATE for a map not initialised); null n_parts or parts with count > 0; n_parts[k] < 0 or
 * > GG_MAX_CLOUD_PARTS; scans[k].n_points other than the sum of its parts' n_points; per part the layout rules of
 * gg_upload_cloud_msg (the error text names the scan and the part). */
int gg_run_merged_cloud_msgs_to_device(gg_handle h, int count, const gg_scan_desc* scans, const int* n_parts,
                                       const gg_cloud_part* parts, const gg_scan_outputs* outs, unsigned select,
                                       int32_t* dev_counts, void* stream);

/* The host-memory form, as gg_upload_cloud_msg is for gg_run_cloud_msgs_to_device: the n_parts payloads in HOST memory
 * are copied to the device, unpacked and transformed into the slot's cloud buffer back to back (part p from record
 * sum(n_points of the parts before p) on).  Follow with gg_run_scans for n_points = the sum of the parts' n_points.
 * GG_E_ARG: slot out of range, n_parts < 0 or > GG_MAX_CLOUD_PARTS, null parts with n_parts > 0, more points than the
 * capacity, a part breaking the layout rules of gg_upload_cloud_msg (the error text names the part). */
int gg_upload_cloud_msgs(gg_handle h, int slot, int n_parts, const gg_cloud_part* parts);
int gg_terrain_image(gg_handle h, int slot, float* dst);
/* The other branch of publish_grid_map_layer (src/GroundGridNodelet.cpp:238-245): the single-channel 8-bit image that
 * grid_map::GridMapCvConverter::toImage<unsigned char, 1>(map, layer, CV_8UC1, img) produces and cv::applyColorMap then
 * colours -- lower / upper = min / max over the finite cells, pixel (i, j) = (uchar)((v - lower) / (upper - lower) * 255),
 * non-finite cells 0.  dst: N*N bytes, row-major (i, j) like the cv::Mat; lower / upper (may be NULL) receive the range.
 * The colour table itself (cv::COLORMAP_TWILIGHT, 256 BGR triples) is OpenCV data: the caller applies it. */
int gg_layer_image_u8(gg_handle h, int slot, const char* name, uint8_t* dst, float* lower, float* upper);

/* The images of publish_grid_map_layer (src/GroundGridNodelet.cpp:216-228,234-291) for `count` distinct slots, written
 * into caller-owned device memory and ordered on the caller's stream: the batched, device-side form of
 * gg_layer_image_u8 / gg_terrain_image.
 *   slots      : `count` distinct slots, each with an initialised map
 *   names      : `n_names` (<= 12) distinct layer names, resolved as in gg_get_layers_to_device ("points" per slot)
 *   dst        : gg_layer_images_to_device: uint8[count][n_names][N][N], the image of scan k and name l at
 *                (k * n_names + l) * N*N, row-major like the cv::Mat of gg_layer_image_u8 (pixel (i, j) at i*N + j);
 *                gg_terrain_images_to_device: float[count][N][N][3] (4-byte aligned), each image that of gg_terrain_image
 *   dev_range  : NULL or float[count][n_names][2] (4-byte aligned): lower, upper of each image
 *   stream     : cudaStream_t; NULL is the legacy default stream.  The contract of gg_get_layers_to_device: the work
 *                starts after everything already enqueued on `stream` and on the stream group of every slot in the
 *                batch, work enqueued on `stream` afterwards sees the images complete, and nothing waits on the host
 *                except the flow control of the parameter staging ring.
 * Pixels and ranges are bit-identical to gg_layer_image_u8 / gg_terrain_image of the same slot and name at the same
 * point of the slot's stream (ordered min / max: -0 below +0; 0 for a non-finite cell; 0 everywhere for a plane that is
 * constant or has no finite cell).
 * count == 0 or n_names == 0 enqueues nothing and returns GG_OK.  Rejected with nothing enqueued: what
 * gg_get_layers_to_device rejects, and (GG_E_ARG) a misaligned dev_range, dst or dev_range overlapping the handle's
 * layers or each other.  gg_terrain_images_to_device without GG_FLAG_FULL_LAYERS: GG_E_LAYER. */
int gg_layer_images_to_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, uint8_t* dst,
                              float* dev_range, void* stream);
int gg_terrain_images_to_device(gg_handle h, int count, const int* slots, float* dst, void* stream);
/* Evaluation tallies (scripts/eval_groundpoint_classifier.py:95-118): the ground-truth SemanticKITTI id of each point
 * travels in `ring` (scripts/kitti_data_publisher.py:117-150); per id, the points predicted ground (49) and non-ground
 * (99).  Absent points (label 0) and ids >= GG_EVAL_IDS are not counted.  gg_eval_accumulate adds the last completed
 * scan of `slot` into one tally of the handle, uint64[GG_EVAL_IDS][2]; gg_eval_read synchronises the handle and copies
 * it out (reset != 0: then zeroes it). */
#define GG_EVAL_IDS 1024
int gg_eval_accumulate(gg_handle h, int slot);
int gg_eval_read(gg_handle h, uint64_t* counts, int reset);

/* The tallies of gg_eval_accumulate for `count` distinct slots, each added into its own tally in caller-owned device
 * memory and ordered on the caller's stream: the batched, device-side form of gg_eval_accumulate + gg_eval_read.
 *   slots      : `count` distinct slots, each with a completed scan (not stopped early)
 *   dev_counts : uint64[count][GG_EVAL_IDS][2] on the handle's device, 8-byte aligned.  The tallies of the last scan of
 *                slots[k] are ADDED to dev_counts[k][id][c], c = 0 for points predicted ground, 1 for non-ground: zero
 *                the buffer once and it keeps running sums per slot over a whole sequence.
 *   stream     : cudaStream_t; NULL is the legacy default stream.  The contract of gg_get_layers_to_device: the work
 *                starts after everything already enqueued on `stream` and on the stream group of every slot in the
 *                batch, work enqueued on `stream` afterwards sees the tallies complete, and nothing waits on the host
 *                except the flow control of the parameter staging ring.
 * The ground truth is read where the scan took its input from:
 *   - gg_filter_cloud, gg_upload_points / gg_upload_cloud_msg + gg_run_scans, gg_run_cloud_msgs_to_device: the slot's
 *     own buffer (a gg_run_cloud_msgs_to_device payload may already be freed);
 *   - gg_filter_cloud_batch: the handle's staging of that batch;
 *   - gg_run_scans_device / gg_run_scans_to_device: the CALLER's cloud, which must still hold the scan's records when
 *     the tallies run (e.g. freed on `stream` only after this call).
 * The tallies are bit-identical to gg_eval_accumulate + gg_eval_read of the same slots at the same point of the slots'
 * streams.  Because `ring` carries the label, a configuration with max_ring below the largest id of interest drops
 * those points from the map (the reference does the same under its KITTI player), but they are still tallied.
 * count == 0 enqueues nothing and returns GG_OK.  Rejected with nothing enqueued:
 *   GG_E_ARG   null handle, slots or dev_counts; count > n_slots; a slot out of range or repeated; dev_counts not
 *              8-byte aligned or overlapping the handle's layers
 *   GG_E_STATE a slot whose map is not initialised, or with no completed scan (none since gg_init_map, or the last
 *              one stopped early)
 * As for every call: a gg_filter_cloud_batch_begin batch that touches the same slots needs a gg_synchronize (or its
 * _wait) first. */
int gg_eval_counts_to_device(gg_handle h, int count, const int* slots, uint64_t* dev_counts, void* stream);

/* Caller-owned DEVICE destinations of one slot of gg_point_info_to_device (on the handle's device; each may be NULL).
 * n = the point count of the slot's last scan (gg_last_scan_points). */
typedef struct gg_point_info {
    uint32_t* codes;   /* [n], 4-byte aligned: class << 24 | cell, bit-identical to gg_get_point_classes */
    float* height;     /* [n], 4-byte aligned: z - ground[cell] */
} gg_point_info;

/* Per-point class and height above the terrain of the last completed scan of `count` distinct slots, written into
 * caller-owned device memory and ordered on the caller's stream: the batched, device-side form of gg_get_point_classes,
 * plus the quantity the label rule compares against its tolerance (src/GroundSegmentation.cpp:171-173).
 *   codes  : for every input point, in input order (for a merged scan: part order), the word gg_get_point_classes returns
 *            for it at the same point of the slot's stream: class << 24 | cell with class 0 absent, 1 kept, 2 kept
 *            (border cell), 3 ignored (ring > max_ring or near range), 4 ignored (border cell), 5 below-ground outlier
 *            (labelled ground) -- the point_index / ignored / outliers lists of insert_cloud (:112-117)
 *   height : for a point with a cell (classes 1-5), __fsub_rn(z, ground[cell]) in fp32, bit-identical to
 *            np.float32(z) - np.float32(G[cell]).  z is the map-frame z the scan rasterized (after any unpack and
 *            transform); G is the "ground" plane at the point of the slot's stream where the call runs: after the scan's
 *            spiral, or what a later gg_set_layer[s_from_device] wrote.  Border and outlier points get heights too (an
 *            outlier's is typically negative).  Absent points get the quiet NaN 0x7fc00000 (as gg_sample_layers_to_device
 *            outside the map).
 *   stream : cudaStream_t; NULL is the legacy default stream.  The contract of gg_get_layers_to_device: the work starts
 *            after everything already enqueued on `stream` and on the stream group of every slot in the batch, work
 *            enqueued on `stream` afterwards sees the outputs, and nothing waits on the host except the flow control of
 *            the parameter staging ring.  The slot's next roll or scan, enqueued after the call, does not change them.
 *            The first call on a handle also allocates the staging of the destinations (cudaMalloc, cudaHostAlloc).
 * Nothing is read from the caller's cloud or payload: both values come from the handle's per-point state and layers.  So,
 * unlike gg_eval_counts_to_device, the call works after gg_run_cloud_msgs_to_device, gg_run_merged_cloud_msgs_to_device
 * or gg_run_scans_to_device with the input already freed, and after gg_filter_cloud_batch with host-packed clouds.
 * count == 0, or a batch with nothing to write (every n == 0 or both pointers NULL), enqueues nothing and returns GG_OK.
 * Rejected with nothing enqueued:
 *   GG_E_ARG   null handle, slots or outs; count > n_slots; a slot out of range or repeated; a misaligned output; an
 *              output range overlapping the handle's layers or another output range of the call (the slots run
 *              concurrently)
 *   GG_E_STATE a slot whose map is not initialised, with no completed scan (none since gg_init_map, or the last one
 *              stopped early), or whose map moved since that scan: a roll with a nonzero cell shift moves every cell
 *              index, so the codes would no longer address the terrain the scan saw.  A roll that does not move is fine.
 * As for every call: a gg_filter_cloud_batch_begin batch that touches the same slots needs a gg_synchronize (or its
 * _wait) first. */
int gg_point_info_to_device(gg_handle h, int count, const int* slots, const gg_point_info* outs, void* stream);

/* *n_points = the point count of the slot's last scan, completed or stopped early (0 before any scan since gg_init_map).
 * An upload of the next cloud does not change it.  Host state: no device wait.  GG_E_ARG: null handle or n_points, slot
 * out of range. */
int gg_last_scan_points(gg_handle h, int slot, size_t* n_points);

/* Per-kernel CUDA-event timing on the launching stream (bench.py roofline).  While enabled every
 * kernel launch is bracketed by an event pair; gg_profile_read synchronises and returns the
 * accumulated milliseconds and launch counts per kernel id (arrays of gg_profile_kernel_count()). */
int gg_profile_enable(gg_handle h, int on);
int gg_profile_read(gg_handle h, double* ms_per_kernel, uint32_t* launches_per_kernel, int reset);
int gg_profile_kernel_count(void);
const char* gg_profile_kernel_name(int id);

/* Output cloud of the last scan of a slot in the reference's order (see gg_filter_cloud). */
int gg_get_output(gg_handle h, int slot, uint32_t* index_out, gg_point* cloud_out, size_t* n_out);

/* Layer access (grid_map::GridMap::operator[] / get(), e.g. GroundSegmentation.cpp:76-78):
 * names "points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight", "variance"
 * always; "groundCandidates", "planeDist", "m2", "meanVariance", "pointsRaw" with
 * GG_FLAG_FULL_LAYERS.  dst/src: N*N floats, column-major.  "expectedPoints" reads the
 * table of GroundSegmentation::init. */
int gg_get_layer(gg_handle h, int slot, const char* name, float* dst);
int gg_set_layer(gg_handle h, int slot, const char* name, const float* src);

/* Raw device pointer of a layer (for NCCL broadcast of the rolling terrain prior: "ground" and
 * "groundpatch" of one slot are contiguous, 2*N*N floats starting at "ground"). */
int gg_layer_device_ptr(gg_handle h, int slot, const char* name, void** dptr);
int gg_set_map_position(gg_handle h, int slot, double x, double y);

/* Layers of `count` distinct slots copied into (get) or out of (set) ONE caller-owned device buffer, ordered on the
 * caller's stream: the batched, device-side form of gg_get_layer / gg_set_layer.
 *   slots      : `count` distinct slots, each with an initialised map
 *   names      : `n_names` (<= 12) distinct layer names, resolved as gg_get_layer resolves them ("points" per slot:
 *                the kept-point count after a scan stopped before labelling, else the non-ground count)
 *   dst / src  : float[count][n_names][N*N] on the handle's device, 4-byte aligned; the plane of scan k and name l
 *                starts at (k * n_names + l) * N*N and is column-major like gg_get_layer (cell (i, j) at i + j*N)
 *   stream     : cudaStream_t; NULL is the legacy default stream.  The same contract as gg_run_scans_to_device: the copy
 *                starts after everything already enqueued on `stream` and on the stream group of every slot in the
 *                batch (so it reads / overwrites the state after the slot's last enqueued scan or roll), and work
 *                enqueued on `stream` after the call sees it complete.  Only the stream groups with slots in the batch
 *                take part; nothing waits on the host except the flow control of the parameter staging ring.  A
 *                stream-ordered allocator may therefore free `src` or reuse `dst` on `stream` right after the call.
 * Later scans of a slot read what gg_set_layers_from_device wrote.  Moving a stream to another slot, handle or GPU:
 * gg_init_map at the old slot's map position, gg_set_slot_config with its configuration, then import "ground" and
 * "groundpatch" (the only layers a scan reads from the previous one): the slot then continues bit-identically.
 * count == 0 or n_names == 0 enqueues nothing and returns GG_OK.  Rejected with nothing enqueued:
 *   GG_E_ARG   null handle; null slots / names / buffer; count > n_slots; a slot out of range or repeated; a name
 *              repeated; n_names > 12; a buffer not 4-byte aligned or overlapping the handle's layers (e.g. a
 *              gg_layer_device_ptr address); on import, "points" together with the layer it names for a slot
 *   GG_E_LAYER an unknown name, a GG_FLAG_FULL_LAYERS layer without the flag, "expectedPoints" (not a slot layer)
 *   GG_E_STATE a slot whose map is not initialised
 * As for every call: a gg_filter_cloud_batch_begin batch that touches the same slots needs a gg_synchronize (or its
 * _wait) first. */
int gg_get_layers_to_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, float* dst, void* stream);
int gg_set_layers_from_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, const float* src,
                              void* stream);

/* Terrain lookups: the values of layers of `count` distinct slots at arbitrary map-frame positions (a planner's samples,
 * another sensor's detections, the points of the next cloud), written into caller-owned device memory and ordered on
 * the caller's stream -- what grid_map's getIndex followed by a layer read gives a consumer of the published map
 * (GroundGridNodelet.cpp:211-214), without exporting whole planes.
 *   slots      : `count` distinct slots, each with an initialised map (no scan needed: the prior after gg_init_map or
 *                after a roll is a valid terrain).  The map position used is the slot's position after its last
 *                enqueued roll (what gg_get_map_position returns at the time of the call).
 *   queries    : queries[k] is the set of positions of slots[k] and where its results go; all DEVICE memory on the
 *                handle's device:
 *                  data       n records of point_step bytes, 4-byte aligned (NULL allowed when n == 0)
 *                  n          <= INT32_MAX, independent of the handle's max_points
 *                  point_step multiple of 4, >= 8: 32 for gg_point records, 8 for float32 [n, 2], 16 for [n, 4] ...
 *                  off_x/y    byte offsets of float32 x, y in the MAP frame; multiples of 4, off + 4 <= point_step
 *                  dst        float32 [n_names][n], 4-byte aligned: the value of name l at query q lands at dst[l*n + q]
 *                  cell       NULL or int32 [n], 4-byte aligned: i + j*N of the query's cell, -1 outside the map
 *   names      : `n_names` (<= 12) distinct layer names, resolved as in gg_get_layers_to_device ("points" per slot)
 *   mode       : GG_SAMPLE_NEAREST or GG_SAMPLE_LINEAR
 *   stream     : cudaStream_t; NULL is the legacy default stream.  The contract of gg_get_layers_to_device: the work
 *                starts after everything already enqueued on `stream` and on the stream group of every slot in the
 *                batch, work enqueued on `stream` afterwards sees the results, and nothing waits on the host except the
 *                flow control of the parameter staging ring.  A stream-ordered allocator may therefore free the
 *                position sets, or reuse their memory, on `stream` right after the call; the slot's next scan, enqueued
 *                after the call, does not change what the call reads.
 * Cell: the rasterizer's own arithmetic (a query lands in exactly the cell a scan point at the same position would):
 * (x, y) widened to double, (i, j) = grid_map getIndexFromPosition (fp64 division, truncation toward zero); the query
 * is inside when checkIfPositionWithinMap holds and 0 <= i, j < N.  Border cells (i or j >= N-3) are ordinary cells
 * here: their value is what the layer holds.  A query outside the map, NaN and +-inf coordinates included, gets
 * cell = -1 and NaN (0x7fc00000) for every name: grid_map throws there, one bad query must not fail a batch.
 * GG_SAMPLE_NEAREST: value = plane[i + j*N], bits unchanged (NaN payloads and -0 included).
 * GG_SAMPLE_LINEAR: this project's own definition (not a restatement of grid_map's atPosition(INTER_LINEAR)).  All
 * arithmetic is fp64, correctly rounded, without contraction:
 *   - the centre of cell (i, j) is grid_map's getPositionFromIndex: off = half - 0.5*res (half = N*res / 2),
 *     cx = (px + off) + res*(double)(-i), cy likewise with j and py;
 *   - neighbour direction si = (x >= cx) ? -1 : +1 (i grows toward -x), sj = (y >= cy) ? -1 : +1;
 *   - fractions tx = |x - cx| / res, ty = |y - cy| / res;
 *   - if i + si or j + sj is outside [0, N), the result is the nearest value;
 *   - otherwise, with a = (i, j), b = (i+si, j), c = (i, j+sj), d = (i+si, j+sj):
 *     v = (((1-tx)(1-ty)*fa + tx(1-ty)*fb) + (1-tx)ty*fc) + tx*ty*fd, each weight rounded once, the sum taken left to
 *     right, and (float)v stored.
 *   Non-finite cells propagate as IEEE arithmetic gives (a zero weight times inf is NaN); a NaN result is stored as
 *   0x7fc00000.
 * count == 0, n_names == 0, or sets that are all empty (n == 0) enqueue nothing and return GG_OK.  Rejected with
 * nothing enqueued (the error text names the set):
 *   GG_E_ARG   what gg_get_layers_to_device rejects for slots and names; null queries; an unknown mode; per set a null
 *              data or dst with n > 0, n > INT32_MAX, a point_step that is not a multiple of 4 or below 8, offsets that
 *              are negative, not multiples of 4 or do not fit point_step, a misaligned data / dst / cell; an output
 *              range (dst, cell) overlapping the handle's layers, any set's positions or another output range (the
 *              sets of different slots run concurrently)
 *   GG_E_LAYER an unknown name, a GG_FLAG_FULL_LAYERS layer without the flag, "expectedPoints"
 *   GG_E_STATE a slot whose map is not initialised */
#define GG_SAMPLE_NEAREST 0
#define GG_SAMPLE_LINEAR 1
typedef struct gg_positions {
    const void* data;
    size_t n;
    int point_step;
    int off_x, off_y;
    float* dst;
    int32_t* cell;
} gg_positions;
int gg_sample_layers_to_device(gg_handle h, int count, const int* slots, const gg_positions* queries, int n_names, const char* const* names,
                               int mode, void* stream);

/* Streams.  Slots are bound to the handle's streams in contiguous groups (GG_STREAMS env,
 * default 4, capped by n_slots; 1 when the caller supplied a stream) and everything that
 * touches a slot is enqueued on its stream.  gg_stream() is the primary stream;
 * gg_fork_streams() makes all streams wait for work already enqueued on it and
 * gg_join_streams() makes it wait for all others, so an event pair recorded on gg_stream()
 * around fork ... join brackets the work of every stream. */
void* gg_stream(gg_handle h);
int gg_num_streams(gg_handle h);
int gg_host_pack_threads(gg_handle h);
/* How the last gg_filter_cloud_batch call moved its clouds: info[0] scans repacked on the host,
 * info[1] scans sent as 32-byte records, info[2] / info[3] the H2D bytes of either kind,
 * info[4] host microseconds until the last cloud was enqueued, info[5] until the call returned
 * (synchronous call only), info[6] / info[7] microseconds the packer threads spent packing / waiting
 * for a staging slot (summed over threads), info[8] microseconds the calling thread had nothing to
 * enqueue. */
int gg_last_batch_transfer(gg_handle h, size_t info[9]);
int gg_fork_streams(gg_handle h);
int gg_join_streams(gg_handle h);

/* Counters for bench.py: number of kernel launches issued by this handle so far. */
uint64_t gg_kernel_launches(gg_handle h);

/* Number of levels / visits of the wavefront schedule of the spiral interpolation (diagnostics). */
int gg_spiral_schedule_info(gg_handle h, int* levels, int* visits, int* max_per_level);

#ifdef __cplusplus
}
#endif
#endif /* GROUNDGRID_B200_H */
