// ls::Buffer (laser_slam_b200/csrc/ls_buffer.cuh) built by a plain host compiler against cudart.
//   buffer_check nogpu: every allocation fails (no device); prints "gpu present" and stops when there is one.
//   buffer_check gpu:   growth, no-op reserves, the pinned variant, moves, and a refused 2^50-byte request.
#include <cstdio>
#include <cstring>
#include <utility>

#include "ls_buffer.cuh"

using ls::Buffer;
using ls::PinnedBuffer;

#define CHECK(c)                                                    \
  do {                                                              \
    if (!(c)) {                                                     \
      std::printf("FAILED line %d: %s\n", __LINE__, #c);            \
      return 1;                                                     \
    }                                                               \
  } while (0)

template <class B>
bool empty(const B& b) {
  return b.get() == nullptr && b.capacity() == 0;
}

// What cudaGetLastError reports with no error pending: cudaSuccess, or the runtime's persistent initialisation error
// (no driver or no device), which every runtime call returns.
cudaError_t idle = cudaSuccess;

// A refused request: the error is returned, the buffer is empty, and nothing is left pending in cudaGetLastError.
template <class B>
int check_refused(B& b, size_t need) {
  CHECK(b.reserve(need, need) != cudaSuccess);
  CHECK(empty(b));
  CHECK(cudaGetLastError() == idle);
  return 0;
}

int no_gpu() {
  Buffer<float> d;
  PinnedBuffer<double> h;
  CHECK(empty(d) && empty(h));
  CHECK(d.reserve(0, 0) == cudaSuccess && empty(d));  // need <= capacity: nothing to do
  if (check_refused(d, 1000) || check_refused(h, 16)) return 1;
  Buffer<float> moved(std::move(d));
  CHECK(empty(moved) && empty(d));
  d = std::move(moved);
  CHECK(empty(moved) && empty(d));
  d.reset();
  CHECK(empty(d));
  return 0;
}

int gpu() {
  Buffer<float> d;
  CHECK(d.reserve(100, 128) == cudaSuccess && d.get() && d.capacity() == 128);
  CHECK(cudaMemset(d.get(), 0, 128 * sizeof(float)) == cudaSuccess);
  float* const p = d.get();
  CHECK(d.reserve(128, 4096) == cudaSuccess && d.get() == p && d.capacity() == 128);  // fits: unchanged
  CHECK(d.reserve(129, 200) == cudaSuccess && d.get() && d.capacity() == 200);
  CHECK(cudaMemset(d.get(), 0, 200 * sizeof(float)) == cudaSuccess);

  PinnedBuffer<int> h;
  CHECK(h.reserve(16, 16) == cudaSuccess && h.get() && h.capacity() == 16);
  for (int i = 0; i < 16; ++i) h.get()[i] = i;
  CHECK(cudaMemcpy(d.get(), h.get(), 16 * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess);
  int back[16] = {};
  CHECK(cudaMemcpy(back, d.get(), sizeof(back), cudaMemcpyDeviceToHost) == cudaSuccess);
  CHECK(std::memcmp(back, h.get(), sizeof(back)) == 0);

  float* const q = d.get();
  Buffer<float> moved(std::move(d));
  CHECK(empty(d) && moved.get() == q && moved.capacity() == 200);
  Buffer<float> other;
  CHECK(other.reserve(8, 8) == cudaSuccess);
  other = std::move(moved);  // frees other's array
  CHECK(empty(moved) && other.get() == q && other.capacity() == 200);

  // More than any device holds: cudaMalloc / cudaMallocHost refuse it without allocating.  A refused growth of a
  // non-empty buffer leaves it empty too.
  Buffer<char> big;
  PinnedBuffer<char> big_host;
  if (check_refused(big, (size_t)1 << 50) || check_refused(big_host, (size_t)1 << 50)) return 1;
  if (check_refused(other, ((size_t)1 << 50) / sizeof(float))) return 1;
  CHECK(cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  int rc;
  if (!std::strcmp(argv[1], "nogpu")) {
    int count = 0;
    if (cudaGetDeviceCount(&count) == cudaSuccess && count > 0) {
      std::printf("gpu present\n");
      return 0;
    }
    cudaGetLastError();
    idle = cudaGetLastError();
    rc = no_gpu();
  } else if (!std::strcmp(argv[1], "gpu")) {
    rc = gpu();
  } else {
    return 2;
  }
  if (rc == 0) std::printf("ok\n");
  return rc;
}
