// Seeding for the occupancy oracle (test infrastructure only): the oracle's own source with one more entry point, which
// replaces a map's known voxels by given ones, so an insert after a .bt read has a reference.  Built from
// oracle/occupancy_oracle.cpp itself with the same flags, so a map created by that library is the type seeded here.
#include "../../oracle/occupancy_oracle.cpp"

extern "C" {

// keys: n packed voxel keys, strictly ascending; vals their float log-odds.
void occo_seed(void* h, const uint64_t* keys, const float* vals, int64_t n) {
  Occ* m = static_cast<Occ*>(h);
  m->keys.assign(keys, keys + n);
  m->vals.assign(vals, vals + n);
}

}  // extern "C"
