// Full-tree oracle (test infrastructure only): octomap's OcTree as OcTree::write saves it, restated from the rules of
// DESIGN.md §4b''''''' -- every known voxel set with its float log-odds (updateNode down the key's path), prune() on
// values (isNodeCollapsible / pruneNode), updateInnerOccupancy (getMaxChildLogOdds) and writeData (writeNodesRecurs).
// Input: known voxels (packed keys kx | ky << 16 | kz << 32 and float log-odds), e.g. the occupancy oracle's map.  Built
// with -ffp-contract=off like the other oracles.
#include <cstdint>
#include <cstring>
#include <fstream>
#include <limits>
#include <vector>

namespace {

const int kTreeDepth = 16;

// A node pool stands in for octomap's pointers: a node's children are 8 consecutive slots created together; a slot that
// is not `exists` is a child that does not exist.
struct Tree {
  std::vector<int32_t> child;  // first of the 8 child slots, -1: no children
  std::vector<uint8_t> exists;
  std::vector<float> value;
  double res = 0;
  int64_t size = 0, leaves = 0;
  std::vector<uint8_t> payload;

  bool childExists(int n, int i) const { return child[n] >= 0 && exists[child[n] + i]; }
  bool hasChildren(int n) const { return child[n] >= 0; }
  int newNode() {
    child.push_back(-1);
    exists.push_back(0);
    value.push_back(0.0f);
    return (int)child.size() - 1;
  }
  void insert(uint64_t key, float v) {
    const int k[3] = {(int)(key & 0xffff), (int)((key >> 16) & 0xffff), (int)((key >> 32) & 0xffff)};
    int n = 0;
    for (int d = 0; d < kTreeDepth; ++d) {
      const int b = kTreeDepth - 1 - d;
      const int i = ((k[0] >> b) & 1) | (((k[1] >> b) & 1) << 1) | (((k[2] >> b) & 1) << 2);
      if (child[n] < 0) {
        const int c = (int)child.size();
        for (int j = 0; j < 8; ++j) newNode();
        child[n] = c;
      }
      n = child[n] + i;
      exists[n] = 1;
    }
    value[n] = v;
  }
  // isNodeCollapsible: all 8 children exist, have no children and hold the first child's value (float ==)
  bool isNodeCollapsible(int n) const {
    if (!childExists(n, 0)) return false;
    const int first = child[n];
    if (hasChildren(first)) return false;
    for (int i = 1; i < 8; ++i)
      if (!childExists(n, i) || hasChildren(first + i) || !(value[first + i] == value[first])) return false;
    return true;
  }
  void pruneRecurs(int n, int depth, int max_depth, int* num_pruned) {
    if (depth < max_depth) {
      for (int i = 0; i < 8; ++i)
        if (childExists(n, i)) pruneRecurs(child[n] + i, depth + 1, max_depth, num_pruned);
    } else if (isNodeCollapsible(n)) {  // pruneNode: the node takes the first child's value, the children are deleted
      value[n] = value[child[n]];
      child[n] = -1;
      ++*num_pruned;
    }
  }
  void prune() {
    for (int depth = kTreeDepth - 1; depth > 0; --depth) {
      int num_pruned = 0;
      pruneRecurs(0, 0, depth, &num_pruned);
      if (num_pruned == 0) break;
    }
  }
  // updateInnerOccupancyRecurs: children first, then the node's value is getMaxChildLogOdds
  void updateInnerOccupancy(int n, int depth) {
    if (!hasChildren(n) || depth >= kTreeDepth) return;
    float mx = -std::numeric_limits<float>::max();
    for (int i = 0; i < 8; ++i) {
      if (!childExists(n, i)) continue;
      updateInnerOccupancy(child[n] + i, depth + 1);
      const float l = value[child[n] + i];
      if (l > mx) mx = l;
    }
    value[n] = mx;
  }
  // writeNodesRecurs: the node's value (OcTreeDataNode::writeData), the byte of existing children, then each child
  void writeNodesRecurs(int n) {
    uint8_t bits = 0;
    for (int i = 0; i < 8; ++i)
      if (childExists(n, i)) bits |= (uint8_t)(1u << i);
    uint8_t v[4];
    std::memcpy(v, &value[n], 4);  // little-endian hosts only, as octomap writes the float's bytes
    payload.insert(payload.end(), v, v + 4);
    payload.push_back(bits);
    ++size;
    if (!bits) ++leaves;
    for (int i = 0; i < 8; ++i)
      if (childExists(n, i)) writeNodesRecurs(child[n] + i);
  }
};

}  // namespace

extern "C" {

// The full tree of n known voxels (packed keys, float log-odds) at resolution res.
void* octo_full_from_voxels(const uint64_t* keys, const float* vals, int64_t n, double res) {
  Tree* t = new Tree();
  t->res = res;
  if (n > 0) {
    t->newNode();  // the root
    t->exists[0] = 1;
    for (int64_t j = 0; j < n; ++j) t->insert(keys[j], vals[j]);
    t->prune();
    t->updateInnerOccupancy(0, 0);
    t->writeNodesRecurs(0);
  }
  std::vector<int32_t>().swap(t->child);
  std::vector<uint8_t>().swap(t->exists);
  std::vector<float>().swap(t->value);
  return t;
}
void octo_full_destroy(void* t) { delete static_cast<Tree*>(t); }
// nodes (octomap's size()), leaves, payload bytes
void octo_full_counts(void* tv, int64_t* out) {
  const Tree* t = static_cast<Tree*>(tv);
  out[0] = t->size;
  out[1] = t->leaves;
  out[2] = (int64_t)t->payload.size();
}
void octo_full_payload(void* tv, uint8_t* out) {
  const Tree* t = static_cast<Tree*>(tv);
  if (!t->payload.empty()) std::memcpy(out, t->payload.data(), t->payload.size());
}
// octomap's OcTree::write: AbstractOcTree::write's header, then writeData.  0 on success.
int octo_full_write(void* tv, const char* path) {
  const Tree* t = static_cast<Tree*>(tv);
  std::ofstream s(path, std::ios_base::out | std::ios_base::binary);
  if (!s.is_open()) return -1;
  s << "# Octomap OcTree file\n";
  s << "# (feel free to add / change comments, but leave the first line as it is!)\n#\n";
  s << "id " << "OcTree" << std::endl;
  s << "size " << t->size << std::endl;
  s << "res " << t->res << std::endl;
  s << "data" << std::endl;
  s.write(reinterpret_cast<const char*>(t->payload.data()), (std::streamsize)t->payload.size());
  s.close();
  return s.fail() ? -1 : 0;
}

}  // extern "C"
