// Host-side reader for the libpointmatcher ICP chain YAML the reference loads with
// icp_.loadFromYaml (reference laser_slam/src/laser_track.cpp:14-21,
// laser_slam/src/incremental_estimator.cpp:52-60).  Only the modules of
// laser_slam/configurations/icp_default.yaml are understood; yaml-cpp is not available, so this is a
// small indentation-insensitive "module name / key: value" scanner, enough for that file's grammar.
#include <cctype>
#include <cstdlib>
#include <cstring>
#include <sstream>
#include <string>

#include "../../include/ls_b200.h"

namespace {

std::string trim(const std::string& s) {
  size_t a = 0, b = s.size();
  while (a < b && std::isspace((unsigned char)s[a])) ++a;
  while (b > a && std::isspace((unsigned char)s[b - 1])) --b;
  return s.substr(a, b - a);
}

}  // namespace

// hash32: two rounds of a multiply-xorshift mixer over (index, salt); the oracle restates it (oracle/__init__.py keep_mask)
extern "C" int ls_keep_point(uint32_t index, uint32_t salt, float prob) {
  if (!(prob < 1.0f)) return 1;
  if (!(prob > 0.0f)) return 0;
  uint32_t h = index * 0x9E3779B1u + salt * 0x85EBCA77u + 0x165667B1u;
  h ^= h >> 15; h *= 0x2C1B3C6Du;
  h ^= h >> 12; h *= 0x297A2D39u;
  h ^= h >> 15;
  return (double)h < (double)prob * 4294967296.0 ? 1 : 0;
}

extern "C" int ls_icp_params_from_yaml(const char* yaml_text, ls_icp_params* p) {
  if (!yaml_text || !p) return LS_ERR_ARG;
  ls_icp_default_params(p);
  bool saw_counter = false, saw_diff = false, saw_trim = false, saw_checkers = false;
  std::string section, module;
  std::istringstream in(yaml_text);
  std::string raw;
  while (std::getline(in, raw)) {
    const size_t hash = raw.find('#');
    if (hash != std::string::npos) raw = raw.substr(0, hash);
    std::string line = trim(raw);
    if (line.empty()) continue;
    const bool top_level = !std::isspace((unsigned char)raw[0]) && raw[0] != '-';
    if (!line.empty() && line[0] == '-') line = trim(line.substr(1));
    std::string key = line, val;
    const size_t colon = line.find(':');
    if (colon != std::string::npos) {
      key = trim(line.substr(0, colon));
      val = trim(line.substr(colon + 1));
    }
    if (top_level) {
      section = key;
      module.clear();
      if (section == "transformationCheckers") saw_checkers = true;
      if (section == "errorMinimizer" && !val.empty()) module = val;
      if (section == "matcher" && !val.empty()) module = val;
      if (section == "errorMinimizer" && !val.empty() && val != "PointToPlaneErrorMinimizer") return LS_ERR_ARG;
      continue;
    }
    // module names end in a known suffix and carry no value (or an empty one)
    const bool is_module = val.empty() && (key.find("Matcher") != std::string::npos || key.find("Filter") != std::string::npos ||
                                           key.find("Minimizer") != std::string::npos ||
                                           key.find("Checker") != std::string::npos || key.find("Inspector") != std::string::npos ||
                                           key.find("Logger") != std::string::npos);
    if (is_module) {
      module = key;
      if (section == "matcher" && module != "KDTreeMatcher") return LS_ERR_ARG;
      if (section == "errorMinimizer" && module != "PointToPlaneErrorMinimizer") return LS_ERR_ARG;
      if (section == "outlierFilters") {
        if (module != "TrimmedDistOutlierFilter") return LS_ERR_ARG;
        saw_trim = true;
      }
      if (section == "readingDataPointsFilters" || section == "referenceDataPointsFilters") {
        ++p->unapplied_modules;  // reported, applied by the caller (ls_keep_point / ls_estimate_normals)
        if (section == "referenceDataPointsFilters" && module.find("SurfaceNormal") != std::string::npos && p->reference_normals_knn == 0)
          p->reference_normals_knn = 5;  // libpointmatcher's default knn of the surface-normal filters
      }
      if (module == "CounterTransformationChecker") saw_counter = true;
      if (module == "DifferentialTransformationChecker") saw_diff = true;
      continue;
    }
    if (val.empty()) continue;
    const double num = std::atof(val.c_str());
    if (section == "readingDataPointsFilters" || section == "referenceDataPointsFilters") {
      const bool reading = section == "readingDataPointsFilters";
      if (module == "RandomSamplingDataPointsFilter" && key == "prob" && reading) p->reading_sampling_prob = (float)num;
      if ((module == "SamplingSurfaceNormalDataPointsFilter" || module == "SurfaceNormalDataPointsFilter") && !reading) {
        if (key == "knn") p->reference_normals_knn = (int)num;
        if (key == "ratio") p->reference_sampling_ratio = (float)num;
      }
      continue;
    }
    if (module == "KDTreeMatcher") {
      if (key == "knn" && (int)num != 1) return LS_ERR_ARG;         // only 1-NN is built
      if (key == "epsilon" && num != 0.0) return LS_ERR_ARG;        // only the exact search is built
      if (key == "maxDist") return LS_ERR_ARG;                      // unbounded search only
    } else if (module == "TrimmedDistOutlierFilter") {
      if (key == "ratio") p->trim_ratio = (float)num;
    } else if (module == "CounterTransformationChecker") {
      if (key == "maxIterationCount") p->max_iterations = (int)num;
    } else if (module == "DifferentialTransformationChecker") {
      if (key == "minDiffRotErr") p->min_diff_rot = (float)num;
      if (key == "minDiffTransErr") p->min_diff_trans = (float)num;
      if (key == "smoothLength") p->smooth_length = (int)num;
    }
  }
  if (!saw_trim) p->trim_ratio = 1.0f;  // no outlier filter: every match has weight 1
  if (saw_checkers) {
    p->use_differential = saw_diff ? 1 : 0;
    if (!saw_counter) p->max_iterations = 40;  // libpointmatcher CounterTransformationChecker default
  }
  if (p->max_iterations < 1 || !(p->trim_ratio > 0.f) || p->trim_ratio > 1.f) return LS_ERR_ARG;
  if (p->use_differential && (p->smooth_length < 1 || p->smooth_length > 15)) return LS_ERR_ARG;
  return LS_OK;
}

namespace {

// A filter of the list with libpointmatcher's defaults, except knn 10 / prob 1 / ratio 1: the values the compat
// DataPointsFilters reader has always filled in (oracle/INPUT_FILTERS.md records the difference).
bool filter_defaults(const std::string& name, ls_point_filter* f) {
  std::memset(f, 0, sizeof(*f));
  f->dim = -1;
  f->knn = 10;
  f->prob = 1.0f;
  f->dist = 1.0f;
  f->step = 10;
  f->remove_inside = 1;
  const float box[6] = {-1.f, 1.f, -1.f, 1.f, -1.f, 1.f};
  std::memcpy(f->box, box, sizeof(box));
  f->leaf[0] = f->leaf[1] = f->leaf[2] = 1.0f;
  if (name == "RemoveNaNDataPointsFilter") f->type = LS_PF_REMOVE_NAN;
  else if (name == "MaxDistDataPointsFilter") f->type = LS_PF_MAX_DIST;
  else if (name == "MinDistDataPointsFilter") f->type = LS_PF_MIN_DIST;
  else if (name == "BoundingBoxDataPointsFilter") f->type = LS_PF_BOUNDING_BOX;
  else if (name == "RandomSamplingDataPointsFilter") f->type = LS_PF_RANDOM_SAMPLING;
  else if (name == "FixStepSamplingDataPointsFilter") f->type = LS_PF_FIX_STEP_SAMPLING;
  else if (name == "VoxelGridDataPointsFilter") f->type = LS_PF_VOXEL_GRID;
  else if (name == "SurfaceNormalDataPointsFilter") f->type = LS_PF_SURFACE_NORMAL;
  else if (name == "SamplingSurfaceNormalDataPointsFilter") f->type = LS_PF_SAMPLING_SURFACE_NORMAL;
  else return false;
  return true;
}

// One `key: value` of the current filter; false if the value cannot be honoured.  Keys a filter does not know are
// ignored, as libpointmatcher's own parameter reader does for the ones it does not use.
bool filter_key(ls_point_filter* f, const std::string& key, const std::string& val, int* end_step, double* step_mult) {
  const double v = std::atof(val.c_str());
  switch (f->type) {
    case LS_PF_MAX_DIST:
    case LS_PF_MIN_DIST:
      if (key == "dim") f->dim = (int)v;
      if (key == (f->type == LS_PF_MAX_DIST ? "maxDist" : "minDist")) f->dist = (float)v;
      break;
    case LS_PF_BOUNDING_BOX: {
      static const char* names[6] = {"xMin", "xMax", "yMin", "yMax", "zMin", "zMax"};
      for (int a = 0; a < 6; ++a)
        if (key == names[a]) f->box[a] = (float)v;
      if (key == "removeInside") f->remove_inside = (int)v;
      break;
    }
    case LS_PF_RANDOM_SAMPLING:
      if (key == "prob") f->prob = (float)v;
      break;
    case LS_PF_FIX_STEP_SAMPLING:
      if (key == "startStep") f->step = (int)v;
      if (key == "endStep") *end_step = (int)v;
      if (key == "stepMult") *step_mult = v;
      break;
    case LS_PF_VOXEL_GRID:
      if (key == "vSizeX") f->leaf[0] = (float)v;
      if (key == "vSizeY") f->leaf[1] = (float)v;
      if (key == "vSizeZ") f->leaf[2] = (float)v;
      if (key == "useCentroid" && (int)v != 1) return false;                 // the cell centre is not built
      if (key == "averageExistingDescriptors" && (int)v != 1) return false;  // descriptors are always averaged
      break;
    case LS_PF_SURFACE_NORMAL:
    case LS_PF_SAMPLING_SURFACE_NORMAL:
      if (key == "knn") f->knn = (int)v;
      if (key == "ratio") f->prob = (float)v;
      break;
    default:
      break;
  }
  return true;
}

bool filter_valid(const ls_point_filter& f, int end_step, double step_mult) {
  switch (f.type) {
    case LS_PF_MAX_DIST:
    case LS_PF_MIN_DIST:
      return f.dim >= -1 && f.dim <= 2;
    case LS_PF_BOUNDING_BOX:
      return f.remove_inside == 0 || f.remove_inside == 1;
    case LS_PF_RANDOM_SAMPLING:
    case LS_PF_SAMPLING_SURFACE_NORMAL:
      return f.prob >= 0.f && f.prob <= 1.f;
    case LS_PF_FIX_STEP_SAMPLING:
      // endStep != startStep or stepMult != 1 make libpointmatcher's filter change its step from one call to the next
      return f.step >= 1 && (end_step < 0 || end_step == f.step) && step_mult == 1.0;
    case LS_PF_VOXEL_GRID:
      return f.leaf[0] > 0.f && f.leaf[1] > 0.f && f.leaf[2] > 0.f;
    default:
      return true;
  }
}

}  // namespace

extern "C" int ls_point_filters_from_yaml(const char* yaml_text, ls_point_filter* out, int capacity, int* n_out) {
  if (!yaml_text || !n_out || (out && capacity < 0)) return LS_ERR_ARG;
  *n_out = 0;
  int n = 0;
  ls_point_filter cur;
  bool open = false;
  int end_step = -1;
  double step_mult = 1.0;
  auto close = [&]() -> bool {
    if (!open) return true;
    open = false;
    if (!filter_valid(cur, end_step, step_mult)) return false;
    if (out) {
      if (n >= capacity) return false;
      out[n] = cur;
    }
    ++n;
    return true;
  };
  std::istringstream in(yaml_text);
  std::string raw;
  while (std::getline(in, raw)) {
    const size_t hash = raw.find('#');
    if (hash != std::string::npos) raw = raw.substr(0, hash);
    std::string line = trim(raw);
    while (!line.empty() && line[0] == '-') line = trim(line.substr(1));
    if (line.empty()) continue;
    const size_t colon = line.find(':');
    const std::string key = trim(colon == std::string::npos ? line : line.substr(0, colon));
    std::string val = colon == std::string::npos ? std::string() : trim(line.substr(colon + 1));
    if (key.size() >= 16 && key.compare(key.size() - 16, 16, "DataPointsFilter") == 0) {
      if (!close()) { *n_out = n; return LS_ERR_ARG; }
      if (!filter_defaults(key, &cur)) { *n_out = n; return LS_ERR_ARG; }  // refused by name
      open = true;
      end_step = -1;
      step_mult = 1.0;
      if (!val.empty() && val.front() == '{') {  // inline map: {key: value, key: value}
        val = val.substr(1, val.find('}') == std::string::npos ? std::string::npos : val.find('}') - 1);
        std::istringstream items(val);
        std::string item;
        while (std::getline(items, item, ',')) {
          const size_t c = item.find(':');
          if (c == std::string::npos) continue;
          if (!filter_key(&cur, trim(item.substr(0, c)), trim(item.substr(c + 1)), &end_step, &step_mult)) {
            *n_out = n;
            return LS_ERR_ARG;
          }
        }
      }
      continue;
    }
    if (!open || val.empty()) continue;
    if (!filter_key(&cur, key, val, &end_step, &step_mult)) { *n_out = n; return LS_ERR_ARG; }
  }
  if (!close()) { *n_out = n; return LS_ERR_ARG; }
  *n_out = n;
  return LS_OK;
}
