// Minimal stand-ins for the third-party types that appear in laser_slam's public API
// (reference laser_slam/include/laser_slam/common.hpp:6-20,87-133; SURVEY.md §8b lists the members used).
// They exist ONLY because Eigen, libpointmatcher, GTSAM, minkindr and mincurves are absent from this build
// environment; with the real libraries present these few types are what an adapter would map 1:1
// (INTEGRATION.md).  Header-only, no dependencies.
#ifndef LASER_SLAM_COMPAT_HPP_
#define LASER_SLAM_COMPAT_HPP_

#include <array>
#include <cctype>
#include <cmath>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <istream>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "ls_b200.h"

// ------------------------------------------------------------------------------------------------ curves::Time
namespace curves {
typedef int64_t Time;  // nanoseconds (mincurves)
}

// ------------------------------------------------------------------------------------------------ kindr::minimal
namespace kindr {
namespace minimal {

typedef std::array<double, 3> Position;
typedef std::array<double, 16> Matrix4d;  // column-major, like Eigen::Matrix4d::data()

// double-precision unit quaternion (w, x, y, z), Hamilton convention
class RotationQuaternion {
 public:
  RotationQuaternion() : q_{1, 0, 0, 0} {}
  RotationQuaternion(double w, double x, double y, double z) : q_{w, x, y, z} {}
  double w() const { return q_[0]; }
  double x() const { return q_[1]; }
  double y() const { return q_[2]; }
  double z() const { return q_[3]; }
  std::array<double, 9> getRotationMatrix() const {  // row-major 3x3
    const double w = q_[0], x = q_[1], y = q_[2], z = q_[3];
    return {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
  }
  // SO3::constructAndRenormalize(R): nearest unit quaternion of an approximately orthonormal matrix
  static RotationQuaternion constructAndRenormalize(const std::array<double, 9>& m) {
    double q[4];
    const double t = m[0] + m[4] + m[8];
    if (t > 0) {
      const double s = std::sqrt(t + 1.0) * 2;
      q[0] = 0.25 * s; q[1] = (m[7] - m[5]) / s; q[2] = (m[2] - m[6]) / s; q[3] = (m[3] - m[1]) / s;
    } else if (m[0] > m[4] && m[0] > m[8]) {
      const double s = std::sqrt(1.0 + m[0] - m[4] - m[8]) * 2;
      q[0] = (m[7] - m[5]) / s; q[1] = 0.25 * s; q[2] = (m[1] + m[3]) / s; q[3] = (m[2] + m[6]) / s;
    } else if (m[4] > m[8]) {
      const double s = std::sqrt(1.0 + m[4] - m[0] - m[8]) * 2;
      q[0] = (m[2] - m[6]) / s; q[1] = (m[1] + m[3]) / s; q[2] = 0.25 * s; q[3] = (m[5] + m[7]) / s;
    } else {
      const double s = std::sqrt(1.0 + m[8] - m[0] - m[4]) * 2;
      q[0] = (m[3] - m[1]) / s; q[1] = (m[2] + m[6]) / s; q[2] = (m[5] + m[7]) / s; q[3] = 0.25 * s;
    }
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double sgn = q[0] >= 0 ? 1.0 : -1.0;
    return RotationQuaternion(sgn * q[0] / n, sgn * q[1] / n, sgn * q[2] / n, sgn * q[3] / n);
  }
  RotationQuaternion inverse() const { return RotationQuaternion(q_[0], -q_[1], -q_[2], -q_[3]); }
  RotationQuaternion operator*(const RotationQuaternion& o) const {
    const double* a = q_.data();
    const double* b = o.q_.data();
    RotationQuaternion r(a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                         a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                         a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
                         a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]);
    const double n = std::sqrt(r.q_[0] * r.q_[0] + r.q_[1] * r.q_[1] + r.q_[2] * r.q_[2] + r.q_[3] * r.q_[3]);
    for (double& v : r.q_) v /= n;
    return r;
  }
  Position rotate(const Position& v) const {
    const std::array<double, 9> R = getRotationMatrix();
    return {R[0] * v[0] + R[1] * v[1] + R[2] * v[2], R[3] * v[0] + R[4] * v[1] + R[5] * v[2],
            R[6] * v[0] + R[7] * v[1] + R[8] * v[2]};
  }

 private:
  std::array<double, 4> q_;
};

// T_a_b: maps coordinates of frame b into frame a (reference common.hpp:97-110)
template <typename Scalar>
class QuatTransformationTemplate {
 public:
  typedef RotationQuaternion Rotation;
  typedef kindr::minimal::Position Position;
  QuatTransformationTemplate() : p_{0, 0, 0} {}
  QuatTransformationTemplate(const Rotation& q, const Position& p) : q_(q), p_(p) {}
  const Rotation& getRotation() const { return q_; }
  const Position& getPosition() const { return p_; }
  QuatTransformationTemplate inverse() const {
    const Rotation qi = q_.inverse();
    const Position t = qi.rotate(p_);
    return QuatTransformationTemplate(qi, Position{-t[0], -t[1], -t[2]});
  }
  QuatTransformationTemplate operator*(const QuatTransformationTemplate& o) const {
    const Position t = q_.rotate(o.p_);
    return QuatTransformationTemplate(q_ * o.q_, Position{t[0] + p_[0], t[1] + p_[1], t[2] + p_[2]});
  }
  Matrix4d getTransformationMatrix() const {
    const std::array<double, 9> R = q_.getRotationMatrix();
    Matrix4d T{};
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) T[c * 4 + r] = R[3 * r + c];
      T[12 + r] = p_[r];
    }
    T[15] = 1.0;
    return T;
  }
  // {qw,qx,qy,qz,tx,ty,tz}: the pose layout of the C ABI
  void toArray7(double* out) const {
    out[0] = q_.w(); out[1] = q_.x(); out[2] = q_.y(); out[3] = q_.z();
    out[4] = p_[0]; out[5] = p_[1]; out[6] = p_[2];
  }
  static QuatTransformationTemplate fromArray7(const double* a) {
    return QuatTransformationTemplate(Rotation(a[0], a[1], a[2], a[3]), Position{a[4], a[5], a[6]});
  }

 private:
  Rotation q_;
  Position p_;
};

}  // namespace minimal
}  // namespace kindr

// ------------------------------------------------------------------------------------------------ PointMatcher<float>
// DataPoints memory layout as libpointmatcher: `features` column-major (dim+1) x N, `descriptors` D x N.
template <typename T>
struct PointMatcher {
  struct ConvergenceError : std::runtime_error {
    explicit ConvergenceError(const std::string& m) : std::runtime_error(m) {}
  };
  // 4x4, column-major (Eigen default), data() is what the C ABI takes
  struct TransformationParameters {
    std::array<T, 16> m;
    TransformationParameters() { setIdentity(); }
    void setIdentity() { m.fill(T(0)); m[0] = m[5] = m[10] = m[15] = T(1); }
    T& operator()(int r, int c) { return m[c * 4 + r]; }
    T operator()(int r, int c) const { return m[c * 4 + r]; }
    T* data() { return m.data(); }
    const T* data() const { return m.data(); }
    template <typename S>
    static TransformationParameters cast(const std::array<S, 16>& src) {
      TransformationParameters t;
      for (int i = 0; i < 16; ++i) t.m[i] = static_cast<T>(src[i]);
      return t;
    }
  };
  struct Label {
    std::string text;
    size_t span;
  };
  // column-major dynamic matrix with the few Eigen members laser_slam touches (rows(), cols(), data(), (r,c)).
  // Copies share their storage until one of them is written (copy-on-write): LaserTrack keeps every scan it is handed
  // and a LaserScan travels by value through the reference's interfaces, so a copy must not move 3.6 MB.  view() borrows
  // caller-owned memory without copying (e.g. a pinned staging buffer the driver fills): it is read-only until the
  // first write, which copies.
  struct Matrix {
    std::shared_ptr<std::vector<T>> own;  // null while empty or borrowed
    const T* ext = nullptr;               // borrowed storage
    size_t nrows = 0, count = 0;
    Matrix() {}
    Matrix(size_t r, size_t c) : own(std::make_shared<std::vector<T>>(r * c)), nrows(r), count(r * c) {}
    static Matrix view(const T* p, size_t r, size_t c) {
      Matrix m;
      m.ext = p;
      m.nrows = r;
      m.count = r * c;
      return m;
    }
    size_t rows() const { return nrows; }
    size_t cols() const { return nrows ? count / nrows : 0; }
    size_t size() const { return count; }
    const T* data() const { return ext ? ext : (own ? own->data() : nullptr); }
    T* data() { detach(); return own ? own->data() : nullptr; }
    T& operator()(size_t r, size_t c) { detach(); return (*own)[c * nrows + r]; }
    T operator()(size_t r, size_t c) const { return data()[c * nrows + r]; }
    void resize(size_t r, size_t c) { detach(); if (!own) own = std::make_shared<std::vector<T>>(); nrows = r; count = r * c; own->resize(count); }
    void assign(size_t r, const T* first, const T* last) {
      own = std::make_shared<std::vector<T>>(first, last);
      ext = nullptr;
      nrows = r;
      count = own->size();
    }
    void append(const Matrix& o) {
      detach();
      if (!own) own = std::make_shared<std::vector<T>>();
      own->insert(own->end(), o.data(), o.data() + o.count);
      count = own->size();
    }
    void push_back(T x) {
      detach();
      if (!own) own = std::make_shared<std::vector<T>>();
      own->push_back(x);
      count = own->size();
    }
    void reserve(size_t n) { detach(); if (!own) own = std::make_shared<std::vector<T>>(); own->reserve(n); }
   private:
    void detach() {
      if (ext) {
        own = std::make_shared<std::vector<T>>(ext, ext + count);
        ext = nullptr;
      } else if (own && own.use_count() > 1) {
        own = std::make_shared<std::vector<T>>(*own);
      }
    }
  };
  struct DataPoints {
    Matrix features;     // 4 x N, column-major: x,y,z,1 per point
    Matrix descriptors;  // D x N, column-major
    std::vector<Label> featureLabels, descriptorLabels;
    size_t descriptorDim = 0;
    size_t getNbPoints() const { return features.cols(); }
    bool descriptorExists(const std::string& name) const {
      for (const auto& l : descriptorLabels)
        if (l.text == name) return true;
      return false;
    }
    // row offset of a descriptor inside a descriptor column, or -1
    int descriptorOffset(const std::string& name) const {
      size_t off = 0;
      for (const auto& l : descriptorLabels) {
        if (l.text == name) return (int)off;
        off += l.span;
      }
      return -1;
    }
    void concatenate(const DataPoints& o) {
      if (getNbPoints() == 0) { *this = o; return; }
      if (o.descriptorDim != descriptorDim) throw std::runtime_error("DataPoints::concatenate: descriptor mismatch");
      features.append(o.features);
      descriptors.append(o.descriptors);
    }
    // (re)place a descriptor block of `span` rows (the SurfaceNormal filters add "normals" this way)
    void setDescriptor(const std::string& name, size_t span, const T* block /* span x N */) {
      const size_t n = getNbPoints();
      if (descriptorExists(name)) {
        const size_t off = (size_t)descriptorOffset(name);
        for (size_t i = 0; i < n; ++i)
          for (size_t r = 0; r < span; ++r) descriptors(off + r, i) = block[i * span + r];
        return;
      }
      Matrix nd(descriptorDim + span, n);
      for (size_t i = 0; i < n; ++i) {
        for (size_t r = 0; r < descriptorDim; ++r) nd(r, i) = descriptors(r, i);
        for (size_t r = 0; r < span; ++r) nd(descriptorDim + r, i) = block[i * span + r];
      }
      descriptors = nd;
      descriptorLabels.push_back({name, span});
      descriptorDim += span;
    }
    // convenience: cloud with a 3-row "normals" descriptor
    static DataPoints fromArrays(const T* feat4, const T* normals3, size_t n) {
      DataPoints d;
      d.features.assign(4, feat4, feat4 + 4 * n);
      d.featureLabels = {{"x", 1}, {"y", 1}, {"z", 1}, {"pad", 1}};
      if (normals3) {
        d.descriptors.assign(3, normals3, normals3 + 3 * n);
        d.descriptorLabels = {{"normals", 3}};
        d.descriptorDim = 3;
      }
      return d;
    }
    // the same cloud as a VIEW of caller-owned arrays (no copy; the arrays must outlive every copy of the DataPoints)
    static DataPoints viewOfArrays(const T* feat4, const T* normals3, size_t n) {
      DataPoints d;
      d.features = Matrix::view(feat4, 4, n);
      d.featureLabels = {{"x", 1}, {"y", 1}, {"z", 1}, {"pad", 1}};
      if (normals3) {
        d.descriptors = Matrix::view(normals3, 3, n);
        d.descriptorLabels = {{"normals", 3}};
        d.descriptorDim = 3;
      }
      return d;
    }
  };
  // One device context per process for the stand-ins below (the LaserTrack / IncrementalEstimator classes own theirs).
  static ls_ctx* sharedContext() {
    static ls_ctx* ctx = nullptr;
    if (!ctx && ls_b200_init(0, &ctx) != LS_OK) throw std::runtime_error("ls_b200_init failed: no usable CUDA device");
    return ctx;
  }

  // PointMatcher<T>::Transformation (reference laser_slam/src/laser_track.cpp:33,265,485; common.hpp:140-147):
  // RigidTransformation::compute / checkParameters / correctParameters.
  struct Transformation {
    DataPoints compute(const DataPoints& in, const TransformationParameters& Tr) const {
      DataPoints out = in;
      const int off = in.descriptorOffset("normals");
      const size_t n = in.getNbPoints();
      std::vector<T> nrm(3 * (n ? n : 1));
      const int rc = ls_transform_cloud(sharedContext(), Tr.data(), in.features.data(), off >= 0 ? in.descriptors.data() + off : nullptr,
                                        (int)in.descriptorDim, (int)n, out.features.data(), off >= 0 ? nrm.data() : nullptr);
      if (rc != LS_OK) throw std::runtime_error(std::string("ls_transform_cloud: ") + ls_b200_last_error(sharedContext()));
      if (off >= 0) out.setDescriptor("normals", 3, nrm.data());
      return out;
    }
    bool checkParameters(const TransformationParameters& Tr) const { return ls_check_rigid(Tr.data()) != 0; }
    TransformationParameters correctParameters(const TransformationParameters& Tr) const {
      TransformationParameters o;
      ls_correct_rigid(Tr.data(), o.data());
      return o;
    }
  };
  struct TransformationRegistrarT {
    std::shared_ptr<Transformation> create(const std::string& name) const {
      if (name != "RigidTransformation") throw std::runtime_error("Transformation '" + name + "' is not available");
      return std::make_shared<Transformation>();
    }
  };
  TransformationRegistrarT TransformationRegistrar;
  static PointMatcher& get() {
    static PointMatcher instance;
    return instance;
  }

  // PointMatcher<T>::DataPointsFilters (reference laser_track.cpp:22-30,146): the filter chain of a YAML list, parsed by
  // ls_point_filters_from_yaml and run on the device by ls_filter_cloud (RemoveNaN, Min/MaxDist, BoundingBox,
  // RandomSampling, FixStepSampling, VoxelGrid, SurfaceNormal, SamplingSurfaceNormal; include/ls_b200.h); any other
  // filter name throws.  The result carries the features and, when there are any, the normals (other descriptors are
  // not carried through).
  struct DataPointsFilters {
    std::vector<ls_point_filter> filters;
    DataPointsFilters() {}
    explicit DataPointsFilters(std::istream& in) {
      std::stringstream ss;
      ss << in.rdbuf();
      const std::string text = ss.str();
      int n = 0;
      if (ls_point_filters_from_yaml(text.c_str(), nullptr, 0, &n) != LS_OK ||
          (filters.resize((size_t)n), ls_point_filters_from_yaml(text.c_str(), filters.data(), n, &n)) != LS_OK)
        throw std::runtime_error("DataPointsFilter #" + std::to_string(n) + " is not available");
    }
    void apply(DataPoints& cloud) const {
      if (filters.empty()) return;
      const size_t n = cloud.getNbPoints();
      const int off = cloud.descriptorOffset("normals");
      bool normals = off >= 0;
      for (const ls_point_filter& f : filters)
        normals = normals || f.type == LS_PF_SURFACE_NORMAL || f.type == LS_PF_SAMPLING_SURFACE_NORMAL;
      std::vector<T> feat(4 * (n ? n : 1)), nrm(3 * (n ? n : 1));
      int m = 0;
      const DataPoints& c = cloud;
      const int rc = ls_filter_cloud(sharedContext(), filters.data(), (int)filters.size(), c.features.data(),
                                     off >= 0 ? c.descriptors.data() + off : nullptr, (int)c.descriptorDim, (int)n, feat.data(),
                                     normals ? nrm.data() : nullptr, &m);
      if (rc != LS_OK) throw std::runtime_error(std::string("ls_filter_cloud: ") + ls_b200_last_error(sharedContext()));
      cloud = DataPoints::fromArrays(feat.data(), normals ? nrm.data() : nullptr, (size_t)m);
    }
    static ls_point_filter filter(int type, int knn, float prob) {
      ls_point_filter f;
      std::memset(&f, 0, sizeof(f));
      f.type = type;
      f.knn = knn;
      f.prob = prob;
      return f;
    }
  };

  // PointMatcher<T>::ICP (reference laser_track.cpp:14-21,496; incremental_estimator.cpp:52-60,108): loadFromYaml /
  // setDefault / compute(reading, reference, T0) -> ls_icp_params_from_yaml / ls_icp_register.  The reference cloud
  // must carry a "normals" descriptor (PointToPlaneErrorMinimizer asserts the same upstream).
  struct ICP {
    ls_icp_params params;
    ls_icp_stats last_stats;
    ICP() { setDefault(); }
    void setDefault() {  // ICPChainBase::setDefault() values (SURVEY.md Appendix A.7)
      ls_icp_default_params(&params);
      params.trim_ratio = 0.85f;
      params.min_diff_rot = 0.001f;
      params.min_diff_trans = 0.001f;
      params.smooth_length = 3;
    }
    void loadFromYaml(std::istream& in) {
      std::stringstream ss;
      ss << in.rdbuf();
      if (ls_icp_params_from_yaml(ss.str().c_str(), &params) != LS_OK) throw std::runtime_error("unsupported ICP chain");
    }
    // readingDataPointsFilters / referenceDataPointsFilters of the chain (icp_default.yaml:1-7) run inside compute(), as in
    // libpointmatcher's ICP::compute: deterministic sampling of the reading, normals (+ sampling) of the reference.
    TransformationParameters compute(const DataPoints& reading_in, const DataPoints& reference_in, const TransformationParameters& T0) {
      DataPoints reading = reading_in, reference = reference_in;
      if (params.reading_sampling_prob < 1.0f) {
        DataPointsFilters chain;
        chain.filters.push_back(DataPointsFilters::filter(LS_PF_RANDOM_SAMPLING, 0, params.reading_sampling_prob));
        chain.apply(reading);
      }
      if (params.reference_normals_knn > 0) {
        DataPointsFilters chain;
        chain.filters.push_back(DataPointsFilters::filter(LS_PF_SAMPLING_SURFACE_NORMAL, params.reference_normals_knn,
                                                          params.reference_sampling_ratio));
        chain.apply(reference);
      }
      const int off = reference.descriptorOffset("normals");
      if (off < 0) throw std::runtime_error("PointToPlaneErrorMinimizer: the reference has no 'normals' descriptor");
      TransformationParameters out = T0;
      const int rc = ls_icp_register(sharedContext(), &params, reading.features.data(), (int)reading.getNbPoints(),
                                     reference.features.data(), reference.descriptors.data() + off, (int)reference.descriptorDim,
                                     (int)reference.getNbPoints(), T0.data(), out.data(), &last_stats, nullptr, nullptr, nullptr);
      if (rc == LS_ERR_CONVERGENCE) throw ConvergenceError(ls_b200_last_error(sharedContext()));
      if (rc != LS_OK) throw std::runtime_error(std::string("ls_icp_register: ") + ls_b200_last_error(sharedContext()));
      return out;
    }
  };
};
#ifndef REG
#define REG(name) name##Registrar  // libpointmatcher: PointMatcher::get().REG(Transformation).create("RigidTransformation")
#endif

// ------------------------------------------------------------------------------------------------ gtsam
namespace gtsam {

typedef uint64_t Key;

// The only factor kinds laser_slam builds are ExpressionFactor<SE3> priors and relative-pose factors
// (reference laser_track.cpp:431-458); a graph is therefore a list of ls_factor records.
class NonlinearFactorGraph {
 public:
  void push_back(const ls_factor& f) { factors_.push_back(f); }
  std::set<Key> keys() const {
    std::set<Key> k;
    for (const ls_factor& f : factors_) {
      if (f.type == LS_FACTOR_PRIOR || !f.fix_a) k.insert(f.key_a);
      if (f.type == LS_FACTOR_BETWEEN) k.insert(f.key_b);
    }
    return k;
  }
  bool empty() const { return factors_.empty(); }
  size_t size() const { return factors_.size(); }
  void clear() { factors_.clear(); }
  const ls_factor& at(size_t i) const { return factors_.at(i); }
  const std::vector<ls_factor>& factors() const { return factors_; }

 private:
  std::vector<ls_factor> factors_;
};

class Values {
 public:
  typedef kindr::minimal::QuatTransformationTemplate<double> SE3;
  void clear() { v_.clear(); }
  void insert(Key k, const SE3& T) {
    if (!v_.emplace(k, T).second) throw std::runtime_error("Values::insert: key already exists");
  }
  bool exists(Key k) const { return v_.count(k) != 0; }
  const SE3& at(Key k) const { return v_.at(k); }
  size_t size() const { return v_.size(); }
  bool empty() const { return v_.empty(); }
  std::map<Key, SE3>::const_iterator begin() const { return v_.begin(); }
  std::map<Key, SE3>::const_iterator end() const { return v_.end(); }

 private:
  std::map<Key, SE3> v_;
};

typedef std::set<Key> KeySet;

// noiseModel::Diagonal::Sigmas / Robust::Create(mEstimator::Cauchy::Create(1), Diagonal)  (reference laser_track.cpp:37-64)
namespace noiseModel {
struct Base {
  typedef std::shared_ptr<Base> shared_ptr;
  std::array<double, 6> sigmas{{1, 1, 1, 1, 1, 1}};
  bool cauchy = false;
};
struct Diagonal {
  typedef std::shared_ptr<Base> shared_ptr;
  template <typename V>
  static shared_ptr Sigmas(const V& v) {
    shared_ptr m = std::make_shared<Base>();
    for (int i = 0; i < 6; ++i) m->sigmas[i] = (double)v[i];
    return m;
  }
};
namespace mEstimator {
struct Cauchy {
  typedef std::shared_ptr<Cauchy> shared_ptr;
  double k = 1.0;
  static shared_ptr Create(double k) {
    if (k != 1.0) throw std::runtime_error("only Cauchy(1) is built (reference laser_track.cpp:41,50)");
    return std::make_shared<Cauchy>();
  }
};
}  // namespace mEstimator
struct Robust {
  static Base::shared_ptr Create(const mEstimator::Cauchy::shared_ptr&, const Base::shared_ptr& base) {
    Base::shared_ptr m = std::make_shared<Base>(*base);
    m->cauchy = true;
    return m;
  }
};
}  // namespace noiseModel
typedef noiseModel::Base NoiseModel;

// Expression<SE3> as laser_slam builds them (reference laser_track.cpp:431-458, incremental_estimator.cpp:117-125):
// a trajectory leaf (key), a constant, inverse(leaf | constant), compose(inverse(a), b).  Nothing else is needed by
// ExpressionFactor<SE3>, whose two shapes are the prior Local(meas, T(key)) and the relative pose
// Local(meas, T(a)^-1 T(b)).
template <typename T>
class Expression {
 public:
  enum Form { kLeaf, kConstant, kInverse, kBetween };
  Expression() {}
  explicit Expression(Key k) : form_(kLeaf), key_b_(k) {}
  explicit Expression(const T& value) : form_(kConstant), const_a_(value) {}
  Form form() const { return form_; }
  Key keyA() const { return key_a_; }
  Key keyB() const { return key_b_; }
  bool aIsConstant() const { return a_const_; }
  const T& constant() const { return const_a_; }
  std::set<Key> keys() const {
    std::set<Key> k;
    if (form_ == kLeaf || form_ == kInverse) { if (!(form_ == kInverse && a_const_)) k.insert(key_b_); }
    if (form_ == kBetween) { if (!a_const_) k.insert(key_a_); k.insert(key_b_); }
    return k;
  }
  static Expression inverseOf(const Expression& e) {
    if (e.form_ != kLeaf && e.form_ != kConstant) throw std::logic_error("inverse() of a composite expression is not built");
    Expression r = e;
    r.form_ = kInverse;
    r.a_const_ = e.form_ == kConstant;
    return r;
  }
  static Expression composeOf(const Expression& a_inv, const Expression& b) {
    if (a_inv.form_ != kInverse || b.form_ != kLeaf) throw std::logic_error("compose(): only inverse(a) * leaf(b) is built");
    Expression r;
    r.form_ = kBetween;
    r.a_const_ = a_inv.a_const_;
    r.const_a_ = a_inv.const_a_;
    r.key_a_ = a_inv.key_b_;
    r.key_b_ = b.key_b_;
    return r;
  }

 private:
  Form form_ = kLeaf;
  Key key_a_ = 0, key_b_ = 0;
  bool a_const_ = false;
  T const_a_;
};

template <typename T>
class ExpressionFactor {
 public:
  ExpressionFactor(const noiseModel::Base::shared_ptr& noise, const T& measured, const Expression<T>& e) {
    std::memset(&f_, 0, sizeof(f_));
    f_.robust = noise->cauchy ? 1 : 0;
    for (int i = 0; i < 6; ++i) f_.sigma[i] = noise->sigmas[i];
    measured.toArray7(f_.meas);
    f_.fixed_a[0] = 1.0;
    if (e.form() == Expression<T>::kLeaf) {
      f_.type = LS_FACTOR_PRIOR;
      f_.key_a = f_.key_b = e.keyB();
    } else if (e.form() == Expression<T>::kBetween) {
      f_.type = LS_FACTOR_BETWEEN;
      f_.key_a = e.keyA();
      f_.key_b = e.keyB();
      if (e.aIsConstant()) {
        f_.fix_a = 1;
        e.constant().toArray7(f_.fixed_a);
      }
    } else {
      throw std::logic_error("ExpressionFactor: unsupported expression");
    }
  }
  const ls_factor& record() const { return f_; }
  operator const ls_factor&() const { return f_; }

 private:
  ls_factor f_;
};

// gtsam::Marginals(graph, values).marginalCovariance(key) (reference laser_track.cpp:421-429): a device pose graph is
// built from the factors and values, and ls_pg_marginals returns the 6x6 block of the inverse Hessian.
class Marginals {
 public:
  typedef std::array<double, 36> Matrix6;  // row-major
  Marginals(const NonlinearFactorGraph& graph, const Values& values) {
    if (ls_pg_create(0, &pg_) != LS_OK) throw std::runtime_error("ls_pg_create failed");
    std::vector<Key> keys;
    std::vector<double> poses;
    for (const auto& kv : values) {
      keys.push_back(kv.first);
      double a[7];
      kv.second.toArray7(a);
      poses.insert(poses.end(), a, a + 7);
    }
    std::vector<uint32_t> tracks(keys.size());
    for (size_t i = 0; i < keys.size(); ++i) tracks[i] = (uint32_t)(keys[i] >> 48);  // LaserTrack keys carry the track id
    if (ls_pg_add_poses(pg_, keys.data(), tracks.data(), poses.data(), (int)keys.size()) != LS_OK ||
        ls_pg_add_factors(pg_, graph.factors().data(), (int)graph.size(), nullptr) != LS_OK) {
      const std::string e = ls_pg_last_error(pg_);
      ls_pg_destroy(pg_);
      throw std::runtime_error("Marginals: " + e);
    }
  }
  ~Marginals() { if (pg_) ls_pg_destroy(pg_); }
  Marginals(const Marginals&) = delete;
  Marginals& operator=(const Marginals&) = delete;
  Matrix6 marginalCovariance(Key key) const {
    Matrix6 c;
    if (ls_pg_marginals(pg_, &key, 1, c.data()) != LS_OK) throw std::runtime_error(std::string("Marginals: ") + ls_pg_last_error(pg_));
    return c;
  }
  std::vector<Matrix6> marginalCovariances(const std::vector<Key>& keys) const {  // one device pass for many keys
    std::vector<Matrix6> c(keys.size());
    if (!keys.empty() && ls_pg_marginals(pg_, keys.data(), (int)keys.size(), c[0].data()) != LS_OK)
      throw std::runtime_error(std::string("Marginals: ") + ls_pg_last_error(pg_));
    return c;
  }

 private:
  ls_pg* pg_ = nullptr;
};

// gtsam::ISAM2 as IncrementalEstimator drives it (reference incremental_estimator.cpp:17-20,156-161,258-264,272-289):
// update(new factors, new values[, remove indices]) / update() run ONE Gauss-Newton pass over the whole device graph each,
// calculateEstimate() returns every value.
struct ISAM2Params {
  void setRelinearizeSkip(int) {}
  void setRelinearizeThreshold(double) {}
};
struct ISAM2Result {
  std::vector<size_t> newFactorsIndices;
  ls_pg_stats stats;
  void print(const std::string& = "") const {}
};
class ISAM2 {
 public:
  explicit ISAM2(const ISAM2Params& = ISAM2Params()) {
    if (ls_pg_create(0, &pg_) != LS_OK) throw std::runtime_error("ls_pg_create failed");
  }
  ~ISAM2() { if (pg_) ls_pg_destroy(pg_); }
  ISAM2(const ISAM2&) = delete;
  ISAM2& operator=(const ISAM2&) = delete;
  ISAM2Result update(const NonlinearFactorGraph& new_factors = NonlinearFactorGraph(), const Values& new_values = Values(),
                     const std::vector<size_t>& remove_factor_indices = std::vector<size_t>()) {
    ISAM2Result r;
    std::vector<Key> keys;
    std::vector<double> poses;
    std::vector<uint32_t> tracks;
    for (const auto& kv : new_values) {
      keys.push_back(kv.first);
      tracks.push_back((uint32_t)(kv.first >> 48));
      double a[7];
      kv.second.toArray7(a);
      poses.insert(poses.end(), a, a + 7);
    }
    std::vector<uint64_t> idx(new_factors.size() ? new_factors.size() : 1), rem(remove_factor_indices.begin(), remove_factor_indices.end());
    if ((!keys.empty() && ls_pg_add_poses(pg_, keys.data(), tracks.data(), poses.data(), (int)keys.size()) != LS_OK) ||
        (!rem.empty() && ls_pg_remove_factors(pg_, rem.data(), (int)rem.size()) != LS_OK) ||
        (new_factors.size() && ls_pg_add_factors(pg_, new_factors.factors().data(), (int)new_factors.size(), idx.data()) != LS_OK) ||
        ls_pg_optimize(pg_, 1, &r.stats) < 0)
      throw std::runtime_error(std::string("ISAM2::update: ") + ls_pg_last_error(pg_));
    r.newFactorsIndices.assign(idx.begin(), idx.begin() + new_factors.size());
    return r;
  }
  Values calculateEstimate() const {
    int n = ls_pg_num_poses(pg_);
    std::vector<Key> keys((size_t)(n > 0 ? n : 1));
    std::vector<double> poses(7 * (size_t)(n > 0 ? n : 1));
    ls_pg_get_poses(pg_, keys.data(), poses.data(), &n);
    Values v;
    for (int i = 0; i < n; ++i) v.insert(keys[i], Values::SE3::fromArray7(&poses[7 * (size_t)i]));
    return v;
  }

 private:
  ls_pg* pg_ = nullptr;
};

}  // namespace gtsam

// kindr::minimal::inverse / compose on expressions (minkindr_gtsam; reference laser_track.cpp:442-448)
namespace kindr {
namespace minimal {
template <typename T>
gtsam::Expression<T> inverse(const gtsam::Expression<T>& e) { return gtsam::Expression<T>::inverseOf(e); }
template <typename T>
gtsam::Expression<T> compose(const gtsam::Expression<T>& a, const gtsam::Expression<T>& b) { return gtsam::Expression<T>::composeOf(a, b); }
}  // namespace minimal
}  // namespace kindr

#endif  // LASER_SLAM_COMPAT_HPP_
