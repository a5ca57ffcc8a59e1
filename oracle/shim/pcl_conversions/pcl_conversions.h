// ORACLE / TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Minimal stand-in for <pcl_conversions/pcl_conversions.h> and what it brings in (pcl::PointCloud, the point macros,
// Eigen::Vector3d), so that the reference's src/preprocess.{h,cpp} compile unmodified without PCL, Eigen or ROS.
//
// - fromROSMsg copies each PointCloud2 field into the point member of the same name, reading the member's own type at the
//   field's byte offset (unaligned reads).  Members without a matching field keep their value-initialised 0, as PCL's
//   fromROSMsg leaves a field it finds no match for.
// - <cmath> is included here, as PCL's headers include it: with it and preprocess.h's `using namespace std`, the
//   reference's abs(float) and atan2(float, float) resolve to the float overloads (fabsf, atan2f), as in a ROS build.
// - Eigen::Vector3d has only the members give_feature / plane_judge use; feature extraction is compiled, never run.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <pcl/point_types.h>
#include <sensor_msgs/PointCloud2.h>

#define EIGEN_ALIGN16 alignas(16)
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define PCL_ADD_POINT4D \
    union {             \
        float data[4];  \
        struct {        \
            float x;    \
            float y;    \
            float z;    \
        };              \
    };
#define POINT_CLOUD_REGISTER_POINT_STRUCT(...)

namespace Eigen {
struct Vector3d {
    double v[3] = {0.0, 0.0, 0.0};
    Vector3d() = default;
    Vector3d(double a, double b, double c) : v{a, b, c} {}
    static Vector3d Zero() { return Vector3d(); }
    void setZero() { v[0] = v[1] = v[2] = 0.0; }
    double dot(const Vector3d& o) const { return v[0] * o.v[0] + v[1] * o.v[1] + v[2] * o.v[2]; }
    double norm() const { return std::sqrt(dot(*this)); }
    void normalize() {
        const double n = norm();
        if (n > 0.0) { v[0] /= n; v[1] /= n; v[2] /= n; }
    }
    Vector3d operator-(const Vector3d& o) const { return Vector3d(v[0] - o.v[0], v[1] - o.v[1], v[2] - o.v[2]); }
    struct Row {
        const Vector3d& a;
        double operator*(const Vector3d& b) const { return a.dot(b); }
    };
    Row transpose() const { return Row{*this}; }
    struct Comma {
        Vector3d& d;
        int i;
        Comma& operator,(double x) { if (i < 3) d.v[i++] = x; return *this; }
    };
    Comma operator<<(double x) { v[0] = x; return Comma{*this, 1}; }
};
}  // namespace Eigen

namespace pcl {
template <class T>
struct PointCloud {
    std::vector<T> points;
    uint32_t width = 0, height = 1;
    bool is_dense = true;
    typedef std::shared_ptr<PointCloud> Ptr;
    typedef std::shared_ptr<const PointCloud> ConstPtr;
    size_t size() const { return points.size(); }
    bool empty() const { return points.empty(); }
    void clear() { points.clear(); width = 0; height = 1; }
    void reserve(size_t n) { points.reserve(n); }
    void resize(size_t n) { points.resize(n); width = uint32_t(n); height = 1; }
    void push_back(const T& p) { points.push_back(p); width = uint32_t(points.size()); height = 1; }
    T& operator[](size_t i) { return points[i]; }
    const T& operator[](size_t i) const { return points[i]; }
    T& back() { return points.back(); }
    PointCloud& operator+=(const PointCloud& o) { points.insert(points.end(), o.points.begin(), o.points.end()); width = uint32_t(points.size()); return *this; }
};

namespace shim {
#define FL_SHIM_FIELD(name)                                                                                                  \
    template <class P> auto put_##name(P& p, const uint8_t* s, int) -> decltype((void)p.name) { std::memcpy(&p.name, s, sizeof(p.name)); } \
    template <class P> void put_##name(P&, const uint8_t*, long) {}
FL_SHIM_FIELD(x)
FL_SHIM_FIELD(y)
FL_SHIM_FIELD(z)
FL_SHIM_FIELD(intensity)
FL_SHIM_FIELD(time)
FL_SHIM_FIELD(t)
FL_SHIM_FIELD(ring)
FL_SHIM_FIELD(reflectivity)
FL_SHIM_FIELD(ambient)
FL_SHIM_FIELD(range)
#undef FL_SHIM_FIELD

template <class P>
void put(P& p, const std::string& name, const uint8_t* s) {
    if (name == "x") put_x(p, s, 0);
    else if (name == "y") put_y(p, s, 0);
    else if (name == "z") put_z(p, s, 0);
    else if (name == "intensity") put_intensity(p, s, 0);
    else if (name == "time") put_time(p, s, 0);
    else if (name == "t") put_t(p, s, 0);
    else if (name == "ring") put_ring(p, s, 0);
    else if (name == "reflectivity") put_reflectivity(p, s, 0);
    else if (name == "ambient") put_ambient(p, s, 0);
    else if (name == "range") put_range(p, s, 0);
}
}  // namespace shim

template <class T>
void fromROSMsg(const sensor_msgs::PointCloud2& m, PointCloud<T>& c) {
    const size_t n = size_t(m.width) * m.height;
    c.points.assign(n, T());
    c.width = m.width;
    c.height = m.height;
    for (size_t i = 0; i < n; i++)
        for (const sensor_msgs::PointField& f : m.fields) shim::put(c.points[i], f.name, &m.data[i * m.point_step + f.offset]);
}

// Preprocess::pub_func only; its output is never read
template <class T>
void toROSMsg(const PointCloud<T>& c, sensor_msgs::PointCloud2& m) {
    m.width = uint32_t(c.size());
    m.height = 1;
}
}  // namespace pcl
