// =====================================================================================
// TEST INFRASTRUCTURE ONLY.  C entry points around the UNMODIFIED reference classes.
//
// oracle/build_ref.py compiles, with zero source edits and straight from where they lie,
//     the reference's src/GroundSegmentation.cpp
//     the reference's src/GroundGrid.cpp
// (+ the reference's include/groundgrid/*.h, include/velodyne_pointcloud/point_types.h) against the CPU
// stand-ins of oracle/ref_shim/ (mini Eigen, CPU grid_map::GridMap, ROS/PCL/tf2 message structs) together
// with this file into oracle/_ref/libgg_ref.so.  The library is the *reference's own arithmetic*: every
// float/double/int promotion is whatever the compiler derives from the reference's expressions.  The
// third-party pieces it runs on (Eigen reduction order, grid_map geometry, tf2 point transform) are
// restatements of the published library sources -- see the headers under oracle/ref_shim/.
//
// Used by tests/ (oracle == _ref bit for bit, golden vectors) and by bench.py's CPU legs
// (cpu_baseline.kind = "reference").  Nothing under groundgrid_b200/ may touch it.
//
// Process model: the reference binds function-local `static` references to the layers / size / resolution
// of the FIRST map it sees (GroundSegmentation.cpp:76-78, 203-213, 317-321, 345-351, 400-401, 447-452) and keeps
// a static base_link<-map transform (GroundGrid.cpp:100).  One loaded copy of this library therefore serves
// exactly ONE map; ggr_create() refuses a second handle.  oracle/ref.py loads a private copy of the .so per
// instance (dlopen of a distinct file = fresh statics).
//
// Geometry: GroundGrid hard-codes `const float mResolution = .33f, mDimension = 120.0f` (GroundGrid.h:70-71).
// To run the unmodified class on the other BASELINE geometries the harness overwrites those two members
// through a pointer before the first update() (the only liberty taken; the resulting map size is checked).
// =====================================================================================
#include <groundgrid/GroundGrid.h>
#include <groundgrid/GroundSegmentation.h>

#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>

namespace {

// same layout as oracle/gg_oracle.cpp ggo::Config and include/groundgrid_b200.h gg_config (cfg/GroundGrid.cfg:8-21 order)
struct GgrConfig {
    int point_count_cell_variance_threshold;
    int max_ring;
    double groundpatch_detection_minimum_threshold;
    double distance_factor;
    double minimum_distance_factor;
    double miminum_point_height_threshold;
    double minimum_point_height_obstacle_threshold;
    double outlier_tolerance;
    double ground_patch_detection_minimum_point_count_threshold;
    double patch_size_change_distance;
    double occupied_cells_decrease_factor;
    double occupied_cells_point_count_factor;
    double min_outlier_detection_ground_confidence;
    int thread_count;
};

typedef velodyne_pointcloud::PointXYZIR RefPoint;
static_assert(sizeof(RefPoint) == 32, "PointXYZIR is a 32-byte record (point_types.h:27-33)");

struct SegmentationAccess : groundgrid::GroundSegmentation {
    const grid_map::Matrix& expected() const { return expectedPoints; }  // protected member, GroundSegmentation.h:66
};

struct Ref {
    groundgrid::GroundGrid grid;
    SegmentationAccess seg;
    ros::NodeHandle nh;
    std::shared_ptr<grid_map::GridMap> map;
    groundgrid::GroundGridConfig cfg;
    int n = 0;
    double filter_seconds = 0.0;
};

bool g_created = false;

geometry_msgs::TransformStamped make_tf(const char* parent, const char* child, const double* q_xyzw, const double* t_xyz) {
    geometry_msgs::TransformStamped t;
    t.header.frame_id = parent;
    t.child_frame_id = child;
    t.transform.rotation.x = q_xyzw[0];
    t.transform.rotation.y = q_xyzw[1];
    t.transform.rotation.z = q_xyzw[2];
    t.transform.rotation.w = q_xyzw[3];
    t.transform.translation.x = t_xyz[0];
    t.transform.translation.y = t_xyz[1];
    t.transform.translation.z = t_xyz[2];
    return t;
}

}  // namespace

extern "C" {

// dimension_m is passed to GroundSegmentation::init as size_t like the nodelet does (GroundGridNodelet.cpp:95 passes
// the float mDimension to a `const size_t dimension` parameter), resolution as float.  Returns NULL if this library
// copy already served a map, or if init()'s cell count would differ from the map's (non-integer dimensions).
void* ggr_create(double dimension_m, float resolution) {
    if (g_created) return nullptr;
    auto* r = new Ref();
    const_cast<float&>(r->grid.mResolution) = resolution;
    const_cast<float&>(r->grid.mDimension) = static_cast<float>(dimension_m);
    r->seg.init(r->nh, static_cast<size_t>(r->grid.mDimension), r->grid.mResolution);
    r->n = static_cast<int>(r->seg.expected().rows());
    const int map_n = static_cast<int>(std::round(static_cast<double>(r->grid.mDimension) / static_cast<double>(r->grid.mResolution)));
    if (map_n != r->n) {
        delete r;
        return nullptr;
    }
    r->grid.setConfig(r->cfg);
    r->seg.setConfig(r->cfg);
    g_created = true;
    return r;
}
void ggr_destroy(void* h) { delete static_cast<Ref*>(h); }
int ggr_cells_per_side(void* h) { return static_cast<Ref*>(h)->n; }

void ggr_set_config(void* h, const GgrConfig* c) {
    auto* r = static_cast<Ref*>(h);
    groundgrid::GroundGridConfig& g = r->cfg;
    g.point_count_cell_variance_threshold = c->point_count_cell_variance_threshold;
    g.max_ring = c->max_ring;
    g.groundpatch_detection_minimum_threshold = c->groundpatch_detection_minimum_threshold;
    g.distance_factor = c->distance_factor;
    g.minimum_distance_factor = c->minimum_distance_factor;
    g.miminum_point_height_threshold = c->miminum_point_height_threshold;
    g.minimum_point_height_obstacle_threshold = c->minimum_point_height_obstacle_threshold;
    g.outlier_tolerance = c->outlier_tolerance;
    g.ground_patch_detection_minimum_point_count_threshold = c->ground_patch_detection_minimum_point_count_threshold;
    g.patch_size_change_distance = c->patch_size_change_distance;
    g.occupied_cells_decrease_factor = c->occupied_cells_decrease_factor;
    g.occupied_cells_point_count_factor = c->occupied_cells_point_count_factor;
    g.min_outlier_detection_ground_confidence = c->min_outlier_detection_ground_confidence;
    g.thread_count = c->thread_count;
    // GroundGridNodelet::callbackReconfigure (GroundGridNodelet.cpp:299-302)
    r->grid.setConfig(g);
    r->seg.setConfig(g);
}
void ggr_get_config(void* h, GgrConfig* c) {
    const groundgrid::GroundGridConfig& g = static_cast<Ref*>(h)->cfg;
    c->point_count_cell_variance_threshold = g.point_count_cell_variance_threshold;
    c->max_ring = g.max_ring;
    c->groundpatch_detection_minimum_threshold = g.groundpatch_detection_minimum_threshold;
    c->distance_factor = g.distance_factor;
    c->minimum_distance_factor = g.minimum_distance_factor;
    c->miminum_point_height_threshold = g.miminum_point_height_threshold;
    c->minimum_point_height_obstacle_threshold = g.minimum_point_height_obstacle_threshold;
    c->outlier_tolerance = g.outlier_tolerance;
    c->ground_patch_detection_minimum_point_count_threshold = g.ground_patch_detection_minimum_point_count_threshold;
    c->patch_size_change_distance = g.patch_size_change_distance;
    c->occupied_cells_decrease_factor = g.occupied_cells_decrease_factor;
    c->occupied_cells_point_count_factor = g.occupied_cells_point_count_factor;
    c->min_outlier_detection_ground_confidence = g.min_outlier_detection_ground_confidence;
    c->thread_count = g.thread_count;
}

// GroundGridNodelet::odom_callback -> GroundGrid::update (GroundGridNodelet.cpp:107-112, GroundGrid.cpp:83-147).
// (x, y, z) = odometry position; q/t = lookupTransform("base_link", "map") as quaternion (x,y,z,w) + translation.
// The first call creates the map (initGroundGrid).  Returns 1 if the map moved, 0 if not, 2 on the creating call,
// -1 if the created map does not have the expected cell count.
int ggr_update(void* h, double x, double y, double z, const double* q_xyzw, const double* t_xyz) {
    auto* r = static_cast<Ref*>(h);
    tf2_ros::ggr_tf_table()[{"base_link", "map"}] = make_tf("base_link", "map", q_xyzw, t_xyz);
    auto odom = std::make_shared<nav_msgs::Odometry>();
    odom->header.frame_id = "map";
    odom->pose.pose.position.x = x;
    odom->pose.pose.position.y = y;
    odom->pose.pose.position.z = z;
    const bool first = !r->map;
    grid_map::Position before(0.0, 0.0);
    if (!first) before = r->map->getPosition();
    r->map = r->grid.update(odom);
    if (first) return (r->map->getSize()(0) == r->n && r->map->getSize()(1) == r->n) ? 2 : -1;
    const grid_map::Position& after = r->map->getPosition();
    return (after(0) != before(0) || after(1) != before(1)) ? 1 : 0;
}
void ggr_get_position(void* h, double* xy) {
    auto* r = static_cast<Ref*>(h);
    xy[0] = r->map->getPosition()(0);
    xy[1] = r->map->getPosition()(1);
}
int ggr_get_expected(void* h, float* dst) {
    const grid_map::Matrix& e = static_cast<Ref*>(h)->seg.expected();
    std::memcpy(dst, e.data(), sizeof(float) * (size_t)e.size());
    return 0;
}
int ggr_get_layer(void* h, const char* name, float* dst) {
    auto* r = static_cast<Ref*>(h);
    if (!r->map || !r->map->exists(name)) return -1;
    const grid_map::Matrix& m = (*r->map)[name];
    std::memcpy(dst, m.data(), sizeof(float) * (size_t)m.size());
    return 0;
}
int ggr_set_layer(void* h, const char* name, const float* src) {
    auto* r = static_cast<Ref*>(h);
    if (!r->map || !r->map->exists(name)) return -1;
    grid_map::Matrix& m = (*r->map)[name];
    std::memcpy(m.data(), src, sizeof(float) * (size_t)m.size());  // in place: static references stay valid
    return 0;
}

// GroundGridNodelet::points_callback -> GroundSegmentation::filter_cloud (GroundGridNodelet.cpp:196,
// GroundSegmentation.cpp:50-197).  pts: npts 32-byte PointXYZIR records in the map frame; origin3 = cloudOrigin;
// q/t = mapToBaseTransform = lookupTransform("map", "base_link").  thread_count comes from the config, as shipped.
// Outputs (each may be NULL): labels[npts] = 0 absent / 49 / 99 per INPUT point; out_cloud = the returned cloud
// (reference order, intensity overwritten); out_index[k] = input index of output point k.  The input index
// travels through filter_cloud in the point's unused 4th float (PCL_ADD_POINT4D padding), which the reference
// copies verbatim with the record.  Returns the output cloud size, -1 without a map.  *seconds (may be NULL)
// receives the wall time of the filter_cloud call alone.
long ggr_filter_cloud(void* h, const void* pts, size_t npts, const float* origin3, const double* q_xyzw, const double* t_xyz,
                      uint8_t* labels, void* out_cloud, uint32_t* out_index, double* seconds) {
    auto* r = static_cast<Ref*>(h);
    if (!r->map) return -1;
    pcl::PointCloud<RefPoint>::Ptr cloud(new pcl::PointCloud<RefPoint>);
    cloud->points.resize(npts);
    if (npts) std::memcpy(static_cast<void*>(cloud->points.data()), pts, npts * sizeof(RefPoint));
    for (size_t i = 0; i < npts; ++i) {
        const uint32_t idx = static_cast<uint32_t>(i);
        std::memcpy(&cloud->points[i].data[3], &idx, 4);
    }
    RefPoint origin;
    std::memset(static_cast<void*>(&origin), 0, sizeof(origin));
    origin.x = origin3[0];
    origin.y = origin3[1];
    origin.z = origin3[2];
    const geometry_msgs::TransformStamped mapToBase = make_tf("map", "base_link", q_xyzw, t_xyz);

    const auto t0 = std::chrono::steady_clock::now();
    pcl::PointCloud<RefPoint>::Ptr out = r->seg.filter_cloud(cloud, origin, mapToBase, *r->map);
    const auto t1 = std::chrono::steady_clock::now();
    r->filter_seconds = std::chrono::duration<double>(t1 - t0).count();
    if (seconds) *seconds = r->filter_seconds;

    if (labels) std::memset(labels, 0, npts);
    const size_t nout = out->points.size();
    for (size_t k = 0; k < nout; ++k) {
        RefPoint p = out->points[k];
        uint32_t idx;
        std::memcpy(&idx, &p.data[3], 4);
        if (labels) labels[idx] = static_cast<uint8_t>(p.intensity);
        if (out_index) out_index[k] = idx;
        // the record the reference returns must be the input record with only the intensity replaced
        const RefPoint* in = reinterpret_cast<const RefPoint*>(static_cast<const char*>(pts) + (size_t)idx * sizeof(RefPoint));
        if (std::memcmp(&p.x, &in->x, 12) != 0 || p.ring != in->ring) return -2;
        if (out_cloud) {
            // padding bytes are not part of the value: take them from the caller's record
            char* dst = static_cast<char*>(out_cloud) + k * sizeof(RefPoint);
            std::memcpy(dst, in, sizeof(RefPoint));
            std::memcpy(dst + offsetof(RefPoint, intensity), &p.intensity, 4);
        }
    }
    return static_cast<long>(nout);
}

// Single phases, public in the reference (GroundSegmentation.h:56-62), for known-answer tests.
void ggr_detect_ground_patches(void* h, int section) {
    auto* r = static_cast<Ref*>(h);
    r->seg.detect_ground_patches(*r->map, static_cast<unsigned short>(section));
}
void ggr_detect_ground_patch(void* h, int S, int i, int j) {
    auto* r = static_cast<Ref*>(h);
    if (S == 3)
        r->seg.detect_ground_patch<3>(*r->map, static_cast<size_t>(i), static_cast<size_t>(j));
    else
        r->seg.detect_ground_patch<5>(*r->map, static_cast<size_t>(i), static_cast<size_t>(j));
}
void ggr_interpolate_cell(void* h, int x, int y) {
    auto* r = static_cast<Ref*>(h);
    r->seg.interpolate_cell(*r->map, static_cast<size_t>(x), static_cast<size_t>(y));
}
void ggr_spiral(void* h, const double* q_xyzw, const double* t_xyz) {
    auto* r = static_cast<Ref*>(h);
    r->seg.spiral_ground_interpolation(*r->map, make_tf("map", "base_link", q_xyzw, t_xyz));
}
void ggr_add_layer(void* h, const char* name, double value) { static_cast<Ref*>(h)->map->add(name, value); }
void ggr_grid_index(void* h, double x, double y, int* idx2, int* inside) {
    auto* r = static_cast<Ref*>(h);
    grid_map::Index gi;
    r->map->getIndex(grid_map::Position(x, y), gi);
    idx2[0] = gi(0);
    idx2[1] = gi(1);
    *inside = r->map->isInside(grid_map::Position(x, y)) ? 1 : 0;
}
void ggr_cell_position(void* h, int i, int j, double* xy) {
    auto* r = static_cast<Ref*>(h);
    grid_map::Position p;
    r->map->getPosition(grid_map::Index(i, j), p);
    xy[0] = p(0);
    xy[1] = p(1);
}
}
