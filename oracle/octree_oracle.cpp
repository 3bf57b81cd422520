// Octree oracle (test infrastructure only): octomap's OcTree as writeBinary leaves it, restated from the rules of
// oracle/OCTREE.md -- every known voxel set to its max-likelihood state (toMaxLikelihood), prune(), writeBinaryConst, and
// octomap_to_point_cloud's leaf iteration.  Input: known voxels (packed keys kx | ky << 16 | kz << 32 and float log-odds),
// e.g. the occupancy oracle's map.  Built with -ffp-contract=off like the other oracles.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <vector>

namespace {

const int64_t kKeyMax = 32768;  // octomap's tree_max_val

// A node pool stands in for octomap's pointers:
// a node's children are 8 consecutive slots created together, and a slot with value 0 is a child that does not exist.
const int kTreeDepth = 16;
const int kFree = 1, kOccupied = 2, kInner = 3;  // node values; a leaf holds its max-likelihood state

struct Tree {
  std::vector<int32_t> child;  // first of the 8 child slots, -1: no children
  std::vector<int8_t> val;
  double res = 0;
  int64_t size = 0;  // octomap's size(): every node
  std::vector<uint8_t> payload;
  std::vector<float> centres;  // occupied leaves, x y z 1
  std::vector<uint8_t> depths;

  bool exists(int n, int i) const { return child[n] >= 0 && val[child[n] + i] != 0; }
  bool hasChildren(int n) const { return child[n] >= 0; }
  int newChildren() {
    const int c = (int)child.size();
    child.insert(child.end(), 8, -1);
    val.insert(val.end(), 8, 0);
    return c;
  }
  // updateNode down the key's path, the voxel then set to its max-likelihood state
  void insert(uint64_t key, int state) {
    const int k[3] = {(int)(key & 0xffff), (int)((key >> 16) & 0xffff), (int)((key >> 32) & 0xffff)};
    int n = 0;
    for (int d = 0; d < kTreeDepth; ++d) {
      const int b = kTreeDepth - 1 - d;
      const int i = ((k[0] >> b) & 1) | (((k[1] >> b) & 1) << 1) | (((k[2] >> b) & 1) << 2);
      if (child[n] < 0) {
        const int c = newChildren();
        child[n] = c;
      }
      n = child[n] + i;
      if (val[n] == 0) val[n] = d + 1 < kTreeDepth ? kInner : (int8_t)state;
    }
    val[n] = (int8_t)state;
  }
  bool isNodeCollapsible(int n) const {
    if (!exists(n, 0)) return false;
    const int first = child[n];
    if (hasChildren(first)) return false;
    for (int i = 1; i < 8; ++i)
      if (!exists(n, i) || hasChildren(first + i) || val[first + i] != val[first]) return false;
    return true;
  }
  void pruneRecurs(int n, int depth, int max_depth, int* num_pruned) {
    if (depth < max_depth) {
      for (int i = 0; i < 8; ++i)
        if (exists(n, i)) pruneRecurs(child[n] + i, depth + 1, max_depth, num_pruned);
    } else if (isNodeCollapsible(n)) {  // pruneNode: the node takes the children's value, the children are deleted
      val[n] = val[child[n]];
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
  void writeBinaryNode(int n) {
    uint8_t b[2] = {0, 0};
    for (int i = 0; i < 8; ++i) {
      if (!exists(n, i)) continue;
      const int c = child[n] + i;
      const int bits = hasChildren(c) ? 3 : (val[c] == kOccupied ? 2 : 1);  // bit 2(i%4): free, 2(i%4)+1: occupied
      b[i / 4] |= (uint8_t)(bits << (2 * (i % 4)));
    }
    payload.push_back(b[0]);
    payload.push_back(b[1]);
    for (int i = 0; i < 8; ++i)
      if (exists(n, i) && hasChildren(child[n] + i)) writeBinaryNode(child[n] + i);
  }
  int64_t countNodes(int n) const {
    int64_t s = 1;
    for (int i = 0; i < 8; ++i)
      if (exists(n, i)) s += countNodes(child[n] + i);
    return s;
  }
  // octomap's keyToCoord(key, depth)
  double keyToCoord(int key, int depth) const {
    if (depth == kTreeDepth) return ((double)(key - (int)kKeyMax) + 0.5) * res;
    const double size = res * (double)(1 << (kTreeDepth - depth));
    return (std::floor(((double)key - (double)kKeyMax) / (double)(1 << (kTreeDepth - depth))) + 0.5) * size;
  }
  // leaf_iterator: a stack of (node, depth, centre key), children pushed 7 ... 0; computeChildKey for the keys
  void occupiedLeaves() {
    struct Item {
      int n, depth, k[3];
    };
    std::vector<Item> stack{{0, 0, {(int)kKeyMax, (int)kKeyMax, (int)kKeyMax}}};
    while (!stack.empty()) {
      const Item it = stack.back();
      stack.pop_back();
      if (hasChildren(it.n)) {
        const int off = (int)kKeyMax >> (it.depth + 1);
        for (int i = 7; i >= 0; --i) {
          if (!exists(it.n, i)) continue;
          Item c{child[it.n] + i, it.depth + 1, {0, 0, 0}};
          for (int a = 0; a < 3; ++a) c.k[a] = ((i >> a) & 1) ? it.k[a] + off : it.k[a] - off - (off ? 0 : 1);
          stack.push_back(c);
        }
      } else if (val[it.n] == kOccupied) {
        for (int a = 0; a < 3; ++a) centres.push_back((float)keyToCoord(it.k[a], it.depth));
        centres.push_back(1.0f);
        depths.push_back((uint8_t)it.depth);
      }
    }
  }
};

Tree* make_tree(const uint64_t* keys, const float* vals, int64_t n, double res, float l_occ) {
  Tree* t = new Tree();
  t->res = res;
  if (n > 0) {
    t->child.push_back(-1);  // the root
    t->val.push_back(kInner);
    for (int64_t j = 0; j < n; ++j) t->insert(keys[j], vals[j] >= l_occ ? kOccupied : kFree);
    t->prune();
    t->size = t->countNodes(0);
    t->writeBinaryNode(0);
    t->occupiedLeaves();
  }
  std::vector<int32_t>().swap(t->child);
  std::vector<int8_t>().swap(t->val);
  return t;
}

}  // namespace

extern "C" {

// The pruned octree of n known voxels (packed keys, log-odds) at resolution res, occupied iff log-odds >= l_occ.
void* octo_tree_from_voxels(const uint64_t* keys, const float* vals, int64_t n, double res, float l_occ) {
  return make_tree(keys, vals, n, res, l_occ);
}
void octo_tree_destroy(void* t) { delete static_cast<Tree*>(t); }
// nodes (octomap's size()), payload bytes, occupied leaves
void octo_tree_counts(void* tv, int64_t* out) {
  const Tree* t = static_cast<Tree*>(tv);
  out[0] = t->size;
  out[1] = (int64_t)t->payload.size();
  out[2] = (int64_t)t->depths.size();
}
void octo_tree_payload(void* tv, uint8_t* out) {
  const Tree* t = static_cast<Tree*>(tv);
  if (!t->payload.empty()) std::memcpy(out, t->payload.data(), t->payload.size());
}
void octo_tree_leaves(void* tv, float* centres4, uint8_t* depths) {
  const Tree* t = static_cast<Tree*>(tv);
  if (!t->depths.empty()) {
    std::memcpy(centres4, t->centres.data(), t->centres.size() * sizeof(float));
    std::memcpy(depths, t->depths.data(), t->depths.size());
  }
}
// octomap's writeBinary: the header as writeBinaryConst streams it, then the payload.  0 on success.
int octo_tree_write(void* tv, const char* path) {
  const Tree* t = static_cast<Tree*>(tv);
  std::ofstream s(path, std::ios_base::out | std::ios_base::binary);
  if (!s.is_open()) return -1;
  s << "# Octomap OcTree binary file\n";
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
