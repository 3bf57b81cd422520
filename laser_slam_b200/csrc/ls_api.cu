// C-ABI implementation (include/ls_b200.h): context, device memory, kernel launches.
// There is no CPU fallback anywhere in this file: every entry point needs a live CUDA device.
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ls_b200.h"
#include "ls_kernels.cuh"

using namespace ls;

#define LS_VERSION 100

// Everything one registration needs on the device.  A context owns one workspace per concurrently
// running problem (ls_icp_register_submap_batch); single-problem entry points use workspace 0.
struct Workspace {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev_launch = nullptr;
  int n_cap = 0, m_cap = 0, cells_cap = 0, tab_cap = 0, hist_cap = 0;
  BuildArrays A{};
  BuildState* bs = nullptr;
  float4* rd = nullptr;  // pre-transformed reading
  int* pos = nullptr;
  float4 *vq = nullptr, *vpts = nullptr;                   // certified candidate lists (ls_grid.cuh VLists)
  float* d2 = nullptr;
  int* ids = nullptr;
  float* d2_out = nullptr;
  IcpWork* work = nullptr;
  float* T_hist = nullptr;
  BuildJob* job_host = nullptr;  // pinned; this workspace's slot of the context's job array
  BuildJob* job_dev = nullptr;
  IcpWork* h_work = nullptr;  // pinned host mirrors of the small results
  Grid* h_grid = nullptr;
  IcpProblem hp;              // host copy of this problem's descriptor
  bool stream_dirty = false;  // work (allocation-time clears) was enqueued on this workspace's own stream
};

struct ls_ctx {
  int device = 0;
  int sm_count = 0;
  int icp_ctas = 0;      // co-resident CTAs for the cooperative ICP kernel
  int icp_ctas_max = 0;  // what the device can hold (occupancy x SMs); icp_ctas <= this
  std::string err;
  uint64_t launches = 0;
  std::vector<Workspace*> ws;
  IcpProblem* probs_dev = nullptr;   // [kMaxBatch]
  IcpProblem* probs_host = nullptr;  // pinned
  BuildJob* jobs_dev = nullptr;      // [kMaxBatch]: workspace b stages its build in slot b
  BuildJob* jobs_host = nullptr;     // pinned
  IcpWork* work_pool = nullptr;      // [kMaxBatch] contiguous, so one memset clears a whole batch
  // staging of the entry points that take host clouds (used on workspace 0's stream; ensure_staging)
  float4* reading = nullptr;                               // raw reading
  float4 *ref_stage = nullptr, *ref_nrm_stage = nullptr;  // reference points and normals (scan frame)
  int reading_cap = 0, ref_cap = 0;
  float* nrm_raw = nullptr;                                // raw normals (upload_normals)
  size_t nrm_raw_cap = 0;
  float* T0_dev = nullptr;                                 // 16 floats: ls_transform_cloud's transformation
  // query-sharded registration: this GPU's exchange buffer (shard_count slots + the arrival counter) and the peers'
  unsigned char* xbuf = nullptr;
  unsigned char* xpeer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int shard_rank = 0, shard_count = 1;
  bool xconnected = false;
  unsigned int xflag_base = 0;  // arrivals the earlier registrations consumed from the counter
  // a batch between ls_icp_register_submap_batch_begin and _end: the workspaces are busy
  bool pending = false;
  int pending_batch = 0;
  std::vector<int> pending_n;
  std::vector<float> pending_T0;
  // ring slots (map, slot index) the in-flight batch reads: an asynchronous upload must not overwrite them
  std::vector<std::pair<const ls_map*, int>> pending_slots;
};
constexpr int kMaxBatch = 160;

struct ls_scan_slot {
  float4* pts = nullptr;
  float4* nrm = nullptr;
  int n = 0;
  uint64_t id = 0;
  bool used = false;
  cudaEvent_t ready = nullptr;  // recorded after an asynchronous upload; consumers wait on it
  bool async = false;           // `ready` is meaningful
};

constexpr int kStageRing = 16;  // normals staging buffers of the asynchronous upload path
struct ls_map {
  ls_ctx* ctx = nullptr;
  int capacity = 0, max_pts = 0;
  uint64_t next_id = 1;
  std::vector<ls_scan_slot> slots;
  // asynchronous uploads (ls_map_push_scan_async): own stream, a small ring of raw-normals staging buffers
  cudaStream_t up_stream = nullptr;
  float* stage[kStageRing] = {};
  size_t stage_cap[kStageRing] = {};
  cudaEvent_t stage_free[kStageRing] = {};
  uint64_t n_async = 0;
  // pinned host staging of ls_map_push_scan (pageable caller memory is copied here, the DMA then runs behind the call)
  float* host_stage[kStageRing] = {};
  size_t host_stage_cap[kStageRing] = {};
};

namespace {

int fail(ls_ctx* ctx, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  return code;
}

// the workspaces are single-tenant: nothing that uses them may run between a batch's begin and end
#define BUSY_CHECK(ctx)                                                                                       \
  do {                                                                                                        \
    if ((ctx)->pending) return fail((ctx), LS_ERR_STATE, "a batch is in flight (ls_icp_register_submap_batch_end first)"); \
  } while (0)

#define CU(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (call);                                                                          \
    if (e_ != cudaSuccess)                                                                            \
      return fail(ctx, e_ == cudaErrorMemoryAllocation ? LS_ERR_NOMEM : LS_ERR_CUDA, "%s: %s", #call, \
                  cudaGetErrorString(e_));                                                            \
  } while (0)

#define LAUNCH_CHECK()                                                                          \
  do {                                                                                          \
    ++ctx->launches;                                                                            \
    cudaError_t e_ = cudaGetLastError();                                                        \
    if (e_ != cudaSuccess) return fail(ctx, LS_ERR_CUDA, "kernel launch: %s", cudaGetErrorString(e_)); \
  } while (0)

template <typename T>
int dev_alloc(ls_ctx* ctx, T** p, size_t count) {
  if (*p) cudaFree(*p);
  *p = nullptr;
  CU(cudaMalloc((void**)p, count * sizeof(T)));
  return LS_OK;
}

inline int blocks_for(int n, int threads, int cap) {
  int b = (n + threads - 1) / threads;
  if (b < 1) b = 1;
  return b > cap ? cap : b;
}

int ensure_capacity(ls_ctx* ctx, Workspace* w, int n, int m, int max_cells, int max_iter) {
  if (n > w->n_cap) {
    const int cap = n + n / 8 + 1024;
    int rc;
    if ((rc = dev_alloc(ctx, &w->rd, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->pos, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->d2, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->vq, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->vpts, (size_t)cap * LS_VK))) return rc;
    if ((rc = dev_alloc(ctx, &w->ids, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->d2_out, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.qkey, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.qperm, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.rd_s, (size_t)cap))) return rc;
    w->n_cap = cap;
  }
  if (m > w->m_cap) {
    const int cap = m + m / 8 + 1024;
    int rc;
    if ((rc = dev_alloc(ctx, &w->A.sub_pts, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.sub_nrm, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.srt_pts, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.srt_nrm, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.pkey, (size_t)cap))) return rc;
    // a fine table exists only for a level-0 cell with > leaf_split (>= 16) points; the pool is also capped at
    // ~1.5 GB (cells beyond the pool stay leaves: slower, still exact, flagged in stats.grid_overflow)
    int tcap = cap / 17 + 1024;
    const int tmax = (int)((size_t)1536 * 1024 * 1024 / ((size_t)LS_FB3 * 12));
    if (tcap > tmax) tcap = tmax;
    if ((rc = dev_alloc(ctx, &w->A.tab1, (size_t)tcap * LS_FB3))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.cnt1, (size_t)tcap * LS_FB3))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.tab1_cell, (size_t)tcap))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.qtab_local, (size_t)tcap * LS_FB3))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.qtab_total, (size_t)tcap))) return rc;
    CU(cudaMemsetAsync(w->A.cnt1, 0, (size_t)tcap * LS_FB3 * sizeof(uint32_t), w->stream));
    w->stream_dirty = true;
    w->A.tab_cap = tcap;
    w->tab_cap = tcap;
    w->m_cap = cap;
  }
  if (max_cells > w->cells_cap) {
    int rc;
    if ((rc = dev_alloc(ctx, &w->A.top, (size_t)max_cells + 1))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.cnt0, (size_t)max_cells + 1))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.pyr, (size_t)max_cells / 2 + 4096))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.topmask, (size_t)max_cells + 1))) return rc;
    if ((rc = dev_alloc(ctx, &w->A.qtop_start, (size_t)max_cells + 1))) return rc;
    CU(cudaMemsetAsync(w->A.cnt0, 0, ((size_t)max_cells + 1) * sizeof(uint32_t), w->stream));
    w->stream_dirty = true;
    w->cells_cap = max_cells;
  }
  if (max_iter > w->hist_cap) {
    int rc;
    if ((rc = dev_alloc(ctx, &w->T_hist, (size_t)max_iter * 16))) return rc;
    w->hist_cap = max_iter;
  }
  return LS_OK;
}

// The context's staging for a host reading of n points and a host reference of m points, grown like the workspaces.
int ensure_staging(ls_ctx* ctx, int n, int m) {
  int rc;
  if (n > ctx->reading_cap) {
    const int cap = n + n / 8 + 1024;
    if ((rc = dev_alloc(ctx, &ctx->reading, (size_t)cap))) return rc;
    ctx->reading_cap = cap;
  }
  if (m > ctx->ref_cap) {
    const int cap = m + m / 8 + 1024;
    if ((rc = dev_alloc(ctx, &ctx->ref_stage, (size_t)cap))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->ref_nrm_stage, (size_t)cap))) return rc;
    ctx->ref_cap = cap;
  }
  return LS_OK;
}

struct Resolved {
  float cell;
  int split, max_cells;
};

Resolved resolve(const ls_icp_params* p) {
  Resolved r;
  r.cell = p->cell_size > 0.f ? p->cell_size : 1.0f;
  r.split = p->leaf_split > 0 ? (p->leaf_split < 16 ? 16 : p->leaf_split) : 32;
  r.max_cells = p->max_cells > 0 ? p->max_cells : (1 << 22);
  if (r.max_cells > (1 << 22)) r.max_cells = 1 << 22;  // tile_sums holds 1024 scan tiles
  if (r.max_cells < 64) r.max_cells = 64;
  return r;
}

int check_params(ls_ctx* ctx, const ls_icp_params* p) {
  if (!p) return fail(ctx, LS_ERR_ARG, "null params");
  if (p->max_iterations < 1 || p->max_iterations > 100000) return fail(ctx, LS_ERR_ARG, "max_iterations out of range");
  if (!(p->trim_ratio > 0.f) || p->trim_ratio > 1.f) return fail(ctx, LS_ERR_ARG, "trim_ratio must be in (0,1]");
  if (p->use_differential && (p->smooth_length < 1 || p->smooth_length > kMaxSmooth))
    return fail(ctx, LS_ERR_ARG, "smooth_length must be in [1,%d]", kMaxSmooth);
  return LS_OK;
}

// Stage workspace w's build job (pinned host slot): the sub-map `parts` (device pointers), the initial guess, and --
// when the registration follows -- the reading.
void fill_job(Workspace* w, const Parts& parts, const float* T0_host, const float4* reading_dev, int n) {
  BuildJob& J = *w->job_host;
  J.parts = parts;
  J.bs = w->bs;
  J.A = w->A;
  J.m = parts.offset[parts.n_parts];
  J.n = n;
  J.reading = reading_dev;
  J.rd = w->rd;
  std::memcpy(J.T0, T0_host, sizeof(J.T0));
}

// The spatial hash of `batch` staged jobs (slots jobs_dev[0..batch)): every phase is ONE launch serving all of them
// (grid.y = job).  Enqueued on `st`; nothing synchronises.
int launch_build(ls_ctx* ctx, const BuildJob* jobs_dev, int batch, int m_max, const Resolved& r, cudaStream_t st) {
  const unsigned int B = (unsigned int)batch;
  const int cap = batch > 1 ? ctx->sm_count * 2 : ctx->sm_count * 8;  // blocks per job: the jobs fill the machine together
  const int pb = blocks_for(m_max, 256, cap);
  reset_build_kernel<<<dim3(1, B), 32, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  assemble_kernel<<<dim3(pb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  setup_kernel<<<dim3(1, B), 32, 0, st>>>(jobs_dev, r.cell, r.max_cells, r.split);
  LAUNCH_CHECK();
  count0_kernel<<<dim3(pb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  const int tiles = (r.max_cells + kScanTile - 1) / kScanTile;
  scan_reduce_kernel<<<dim3(tiles, B), kScanThreads, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  scan_apply_kernel<<<dim3(tiles, B), kScanThreads, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  pyramid1_kernel<<<dim3(blocks_for(r.max_cells / 16 + 1, 256, batch > 1 ? ctx->sm_count : ctx->sm_count * 4), B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  pyramid_up_kernel<<<dim3(1, B), 1024, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  count1_kernel<<<dim3(pb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  tables_kernel<<<dim3(cap, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  scatter_kernel<<<dim3(pb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  return LS_OK;
}

// R' = T_refMean_dataIn * R for every staged job, then the readings are ordered by their map's cell keys (q_count_kernel).
int launch_reading_sort(ls_ctx* ctx, const BuildJob* jobs_dev, int batch, int n_max, const Resolved& r, cudaStream_t st) {
  const unsigned int B = (unsigned int)batch;
  const int cap = batch > 1 ? ctx->sm_count * 2 : ctx->sm_count * 8;
  const int qb = blocks_for(n_max, 256, cap);
  const int scan_tiles = (r.max_cells + kScanTile - 1) / kScanTile;
  reading_kernel<<<dim3(qb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  q_count_kernel<<<dim3(qb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  q_tables_kernel<<<dim3(cap, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  q_scan_reduce_kernel<<<dim3(scan_tiles, B), kScanThreads, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  q_scan_apply_kernel<<<dim3(scan_tiles, B), kScanThreads, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  q_scatter_kernel<<<dim3(qb, B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  return LS_OK;
}

// Single problem on workspace w: stage the job (the reading may follow in prep_icp), upload it, build.
int enqueue_build(ls_ctx* ctx, Workspace* w, const Parts& parts, const Resolved& r, const float* T0_host) {
  fill_job(w, parts, T0_host, nullptr, 0);
  CU(cudaMemcpyAsync(w->job_dev, w->job_host, sizeof(BuildJob), cudaMemcpyHostToDevice, w->stream));
  return launch_build(ctx, w->job_dev, 1, w->job_host->m, r, w->stream);
}

int upload_normals(ls_ctx* ctx, Workspace* w, const float* normals, int stride, int n, float4* dst) {
  // the descriptor block may be addressed at a row offset (normals = descriptors.data() + row, stride = D): the last
  // point's normal ends (n-1)*stride + 3 floats after `normals`, and nothing beyond that may be read
  const size_t need = n > 0 ? (stride <= 8 ? (size_t)(n - 1) * (size_t)stride + 3 : (size_t)n * 3) : 0;
  if (need > ctx->nrm_raw_cap) {
    int rc;
    if ((rc = dev_alloc(ctx, &ctx->nrm_raw, need + 4096))) return rc;
    ctx->nrm_raw_cap = need + 4096;
  }
  int dstride = stride;
  if (stride <= 8) {
    CU(cudaMemcpyAsync(ctx->nrm_raw, normals, need * sizeof(float), cudaMemcpyHostToDevice, w->stream));
  } else {
    CU(cudaMemcpy2DAsync(ctx->nrm_raw, 3 * sizeof(float), normals, (size_t)stride * sizeof(float), 3 * sizeof(float),
                         (size_t)n, cudaMemcpyHostToDevice, w->stream));
    dstride = 3;
  }
  expand_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(ctx->nrm_raw, dstride, n, dst);
  LAUNCH_CHECK();
  return LS_OK;
}

// Fill workspace w's problem descriptor for the persistent ICP kernel (host side only).
int fill_problem(ls_ctx* ctx, Workspace* w, const ls_icp_params* prm, int n, const float T0[16], bool want_matches,
                 bool want_hist) {
  IcpProblem& hp = w->hp;
  hp.bs = w->bs;
  hp.view.top = w->A.top;
  hp.view.tab1 = w->A.tab1;
  hp.view.pts = w->A.srt_pts;
  hp.view.pyr = w->A.pyr;
  hp.view.topmask = w->A.topmask;
  hp.nrm = w->A.srt_nrm;
  hp.rd = w->A.rd_s;
  hp.n = n;
  hp.pos = w->pos;
  hp.d2 = w->d2;
  hp.ids = w->ids;
  hp.d2_out = w->d2_out;
  hp.qperm = w->A.qperm;
  hp.lists.vq = w->vq;
  hp.lists.vpts = w->vpts;
  hp.lists.n = n;
  hp.work = w->work;
  hp.shard_rank = 0;
  hp.shard_count = 1;
  std::memset(&hp.link, 0, sizeof(hp.link));
  hp.T_hist = want_hist ? w->T_hist : nullptr;
  if (want_hist) {  // entries past the executed iterations read as zeros, not as stale device memory
    CU(cudaMemsetAsync(w->T_hist, 0, (size_t)prm->max_iterations * 16 * sizeof(float), w->stream));
    w->stream_dirty = true;
  }
  hp.want_matches = want_matches ? 1 : 0;
  hp.phase_ns = nullptr;
  std::memcpy(hp.T0, T0, sizeof(hp.T0));
  return LS_OK;
}

// Single problem: stage the reading in the job built by enqueue_build, sort it, clear the scratch, fill the descriptor.
// Enqueued on the workspace's stream; nothing synchronises.
int prep_icp(ls_ctx* ctx, Workspace* w, const ls_icp_params* prm, const float4* reading_dev, int n, const float T0[16],
             bool want_matches, bool want_hist) {
  w->job_host->reading = reading_dev;
  w->job_host->n = n;
  CU(cudaMemcpyAsync(w->job_dev, w->job_host, sizeof(BuildJob), cudaMemcpyHostToDevice, w->stream));
  int rc;
  if ((rc = launch_reading_sort(ctx, w->job_dev, 1, n, resolve(prm), w->stream))) return rc;
  CU(cudaEventRecord(w->ev1, w->stream));
  CU(cudaMemsetAsync(w->work, 0, sizeof(IcpWork), w->stream));
  return fill_problem(ctx, w, prm, n, T0, want_matches, want_hist);
}

// One cooperative launch over `batch` staged problems (workspaces 0..batch-1): the grid is partitioned into
// `batch` groups of CTAs, each with its own barrier.  Runs on workspace 0's stream after every workspace's
// staging has finished; on return the results are on the host (pinned mirrors).
int launch_icp(ls_ctx* ctx, const ls_icp_params* prm, int batch, int n_max, bool sharded = false) {
  Workspace* w0 = ctx->ws[0];
  for (int b = 0; b < batch; ++b) ctx->probs_host[b] = ctx->ws[b]->hp;
  CU(cudaMemcpyAsync(ctx->probs_dev, ctx->probs_host, sizeof(IcpProblem) * (size_t)batch, cudaMemcpyHostToDevice, w0->stream));
  IcpParamsDev dp;
  dp.max_iterations = prm->max_iterations;
  dp.trim_ratio = prm->trim_ratio;
  dp.use_differential = prm->use_differential;
  dp.min_diff_rot = prm->min_diff_rot;
  dp.min_diff_trans = prm->min_diff_trans;
  dp.smooth_length = prm->smooth_length;
  int ctas = ctx->icp_ctas / batch;   // CTAs per problem; every CTA of the grid must be co-resident
  const int need = (n_max + 31) / 32;
  if (ctas > need) ctas = need;
  if (ctas < 1) ctas = 1;
  const IcpProblem* probs = ctx->probs_dev;
  int dynamic = batch > 1 ? 1 : 0;  // several problems: warps pull work from per-problem counters
  void* args[] = {(void*)&probs, (void*)&ctas, (void*)&dp, (void*)&dynamic};
  if (sharded) {  // narrow the staged problem to this shard's queries (cuts at cell starts, computed on the device)
    shard_slice_kernel<<<1, 32, 0, w0->stream>>>(ctx->probs_dev, w0->job_dev, w0->hp.shard_rank, w0->hp.shard_count);
    LAUNCH_CHECK();
  }
  CU(cudaEventRecord(w0->ev_launch, w0->stream));
  CU(cudaLaunchCooperativeKernel((void*)icp_kernel, dim3(ctas * batch), dim3(kIcpThreads), args, kIcpPairBytes, w0->stream));
  ++ctx->launches;
  CU(cudaEventRecord(w0->ev2, w0->stream));
  for (int b = 0; b < batch; ++b) {
    Workspace* w = ctx->ws[b];
    // only the results at the tail of the scratch come back (not the 48 KB of histograms in front of them)
    constexpr size_t off = offsetof(IcpWork, T_out);
    CU(cudaMemcpyAsync(reinterpret_cast<char*>(w->h_work) + off, reinterpret_cast<const char*>(w->work) + off,
                       sizeof(IcpWork) - off, cudaMemcpyDeviceToHost, w0->stream));
    CU(cudaMemcpyAsync(w->h_grid, &w->bs->grid, sizeof(Grid), cudaMemcpyDeviceToHost, w0->stream));
  }
  return LS_OK;
}

// After launch_icp + a synchronise of workspace 0's stream: unpack one problem's results.
int fetch_icp(ls_ctx* ctx, Workspace* w, int n, const float T0[16], float T_out[16], ls_icp_stats* stats,
              bool batch_timing = false) {
  const IcpWork& wk = *w->h_work;
  std::memcpy(T_out, wk.T_out, 16 * sizeof(float));
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->iterations = wk.iterations;
    stats->converged = wk.converged;
    stats->max_iter_reached = wk.max_iter_reached;
    stats->last_kept = wk.last_kept;
    stats->last_limit = wk.last_limit;
    stats->used_ratio = n > 0 ? (float)wk.last_kept / (float)n : 0.f;
    float ms = 0.f, bms = 0.f, kms = 0.f;
    const Workspace* tw = batch_timing ? ctx->ws[0] : w;  // a batch is staged and built as one: its timing is shared
    cudaEventElapsedTime(&ms, tw->ev0, ctx->ws[0]->ev2);  // staging .. end of the (shared) ICP launch
    cudaEventElapsedTime(&bms, tw->ev0, tw->ev1);
    cudaEventElapsedTime(&kms, ctx->ws[0]->ev_launch, ctx->ws[0]->ev2);
    stats->device_ms = ms;
    stats->build_ms = bms;
    stats->icp_ms = kms;
    stats->grid_cells = w->h_grid->n_cells0;
    stats->grid_tables = w->h_grid->n_tab1;
    stats->grid_overflow = w->h_grid->overflow;
  }
  if (wk.status != 0) {
    std::memcpy(T_out, T0, 16 * sizeof(float));
    return fail(ctx, LS_ERR_CONVERGENCE, "ICP: no point to minimise / non-finite transformation");
  }
  return LS_OK;
}

// single problem: stage on workspace 0, launch, optional arrays, fetch
int run_icp(ls_ctx* ctx, const ls_icp_params* prm, const float4* reading_dev, int n, const float T0[16],
            float T_out[16], ls_icp_stats* stats, int32_t* opt_ids, float* opt_d2, float* opt_T_hist) {
  Workspace* w = ctx->ws[0];
  int rc;
  if ((rc = prep_icp(ctx, w, prm, reading_dev, n, T0, opt_ids || opt_d2, opt_T_hist != nullptr))) return rc;
  if ((rc = launch_icp(ctx, prm, 1, n))) return rc;
  if (opt_ids) CU(cudaMemcpyAsync(opt_ids, w->ids, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, w->stream));
  if (opt_d2) CU(cudaMemcpyAsync(opt_d2, w->d2_out, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  if (opt_T_hist)
    CU(cudaMemcpyAsync(opt_T_hist, w->T_hist, (size_t)prm->max_iterations * 16 * sizeof(float), cudaMemcpyDeviceToHost,
                       w->stream));
  CU(cudaStreamSynchronize(w->stream));
  return fetch_icp(ctx, w, n, T0, T_out, stats);
}

bool is_identity16(const float* T) {
  for (int i = 0; i < 16; ++i)
    if (T[i] != ((i % 5 == 0) ? 1.f : 0.f)) return false;
  return true;
}

const ls_scan_slot* find_slot(const ls_map* map, uint64_t id) {
  const ls_scan_slot& s = map->slots[id % (uint64_t)map->capacity];  // ids are handed out round-robin over the ring
  return (s.used && s.id == id) ? &s : nullptr;
}

// consumers of a slot filled by ls_map_push_scan_async order themselves behind its upload
int wait_slot(const ls_scan_slot* s, cudaStream_t consumer) {
  if (s->async && consumer && cudaStreamWaitEvent(consumer, s->ready, 0) != cudaSuccess) return LS_ERR_CUDA;
  return LS_OK;
}

int make_parts(ls_ctx* ctx, const ls_map* map, int n_parts, const uint64_t* part_ids, const float* T_parts, Parts* out,
               cudaStream_t consumer) {
  if (n_parts < 1 || n_parts > kMaxParts) return fail(ctx, LS_ERR_ARG, "n_parts must be in [1,%d]", kMaxParts);
  Parts& parts = *out;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = n_parts;
  long long off = 0;
  for (int p = 0; p < n_parts; ++p) {
    const ls_scan_slot* s = find_slot(map, part_ids[p]);
    if (!s) return fail(ctx, LS_ERR_STATE, "scan %llu is not resident (evicted or never pushed)",
                        (unsigned long long)part_ids[p]);
    if (wait_slot(s, consumer) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
    parts.offset[p] = (int)off;
    parts.pts[p] = s->pts;
    parts.nrm[p] = s->nrm;
    std::memcpy(parts.T[p], T_parts + 16 * p, 16 * sizeof(float));
    parts.identity[p] = is_identity16(T_parts + 16 * p) ? 1 : 0;
    off += s->n;
    if (off > 0x3fffffff) return fail(ctx, LS_ERR_ARG, "sub-map too large");
  }
  parts.offset[n_parts] = (int)off;
  return LS_OK;
}

}  // namespace

extern "C" {

int ls_b200_version(void) { return LS_VERSION; }

namespace {
Workspace* new_workspace(ls_ctx* ctx, int index) {
  Workspace* w = new Workspace();
  w->work = ctx->work_pool + index;
  w->job_dev = ctx->jobs_dev + index;
  w->job_host = ctx->jobs_host + index;
  bool ok = cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreate(&w->ev0) == cudaSuccess && cudaEventCreate(&w->ev1) == cudaSuccess &&
            cudaEventCreate(&w->ev2) == cudaSuccess && cudaEventCreate(&w->ev_launch) == cudaSuccess &&
            cudaMalloc((void**)&w->bs, sizeof(BuildState)) == cudaSuccess &&
            cudaMallocHost((void**)&w->h_work, sizeof(IcpWork)) == cudaSuccess &&
            cudaMallocHost((void**)&w->h_grid, sizeof(Grid)) == cudaSuccess;
  if (!ok) return nullptr;  // partially built workspace is leaked only on an out-of-memory init failure
  return w;
}
void free_workspace(Workspace* w) {
  if (!w) return;
  if (w->stream) cudaStreamSynchronize(w->stream);
  void* bufs[] = {w->A.sub_pts, w->A.sub_nrm, w->A.srt_pts, w->A.srt_nrm, w->A.pkey, w->A.top, w->A.cnt0, w->A.tab1, w->A.cnt1,
                  w->A.tab1_cell, w->A.pyr, w->A.topmask, w->bs, w->rd, w->pos, w->d2,
                  w->ids, w->vq, w->vpts, w->T_hist, w->d2_out, w->A.qkey, w->A.qperm, w->A.rd_s,
                  w->A.qtab_local, w->A.qtab_total, w->A.qtop_start};
  for (void* b : bufs)
    if (b) cudaFree(b);
  if (w->h_work) cudaFreeHost(w->h_work);
  if (w->h_grid) cudaFreeHost(w->h_grid);
  if (w->ev0) cudaEventDestroy(w->ev0);
  if (w->ev1) cudaEventDestroy(w->ev1);
  if (w->ev2) cudaEventDestroy(w->ev2);
  if (w->ev_launch) cudaEventDestroy(w->ev_launch);
  if (w->stream) cudaStreamDestroy(w->stream);
  delete w;
}
int ensure_workspaces(ls_ctx* ctx, int count) {
  while ((int)ctx->ws.size() < count) {
    Workspace* w = new_workspace(ctx, (int)ctx->ws.size());
    if (!w) return fail(ctx, LS_ERR_NOMEM, "workspace allocation failed");
    ctx->ws.push_back(w);
  }
  return LS_OK;
}
}  // namespace

int ls_b200_init(int device, ls_ctx** out) {
  if (!out) return LS_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return LS_ERR_CUDA;  // no CPU fallback
  if (device < 0 || device >= count) return LS_ERR_ARG;
  ls_ctx* ctx = new ls_ctx();
  ctx->device = device;
  auto bail = [&](int code) {
    ls_b200_destroy(ctx);
    return code;
  };
  if (cudaSetDevice(device) != cudaSuccess) return bail(LS_ERR_CUDA);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return bail(LS_ERR_CUDA);
  if (!prop.cooperativeLaunch) return bail(LS_ERR_CUDA);
  ctx->sm_count = prop.multiProcessorCount;
  int occ = 0;
  if (cudaFuncSetAttribute(icp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kIcpPairBytes) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, icp_kernel, kIcpThreads, kIcpPairBytes) != cudaSuccess || occ < 1)
    return bail(LS_ERR_CUDA);
  ctx->icp_ctas = ctx->icp_ctas_max = occ * ctx->sm_count;
  if (cudaMalloc((void**)&ctx->probs_dev, sizeof(IcpProblem) * kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (cudaMallocHost((void**)&ctx->probs_host, sizeof(IcpProblem) * kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (cudaMalloc((void**)&ctx->jobs_dev, sizeof(BuildJob) * kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (cudaMallocHost((void**)&ctx->jobs_host, sizeof(BuildJob) * kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (cudaMalloc((void**)&ctx->work_pool, sizeof(IcpWork) * kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (cudaMalloc((void**)&ctx->T0_dev, 16 * sizeof(float)) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ensure_workspaces(ctx, 1) != LS_OK) return bail(LS_ERR_NOMEM);
  *out = ctx;
  return LS_OK;
}

void ls_b200_destroy(ls_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (Workspace* w : ctx->ws) free_workspace(w);
  if (ctx->probs_dev) cudaFree(ctx->probs_dev);
  if (ctx->probs_host) cudaFreeHost(ctx->probs_host);
  if (ctx->jobs_dev) cudaFree(ctx->jobs_dev);
  if (ctx->jobs_host) cudaFreeHost(ctx->jobs_host);
  if (ctx->work_pool) cudaFree(ctx->work_pool);
  void* stage[] = {ctx->reading, ctx->ref_stage, ctx->ref_nrm_stage, ctx->nrm_raw, ctx->T0_dev};
  for (void* b : stage)
    if (b) cudaFree(b);
  ls_shard_exchange_close(ctx);
  delete ctx;
}

const char* ls_b200_last_error(const ls_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
uint64_t ls_b200_launch_count(const ls_ctx* ctx) { return ctx ? ctx->launches : 0; }
int ls_b200_set_icp_cta_budget(ls_ctx* ctx, int ctas) {
  if (!ctx || ctas < 0) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  ctx->icp_ctas = (ctas == 0 || ctas > ctx->icp_ctas_max) ? ctx->icp_ctas_max : ctas;
  return LS_OK;
}
int ls_b200_icp_cta_budget(const ls_ctx* ctx) { return ctx ? ctx->icp_ctas : LS_ERR_ARG; }

void ls_icp_default_params(ls_icp_params* p) {
  if (!p) return;
  p->max_iterations = 40;
  p->trim_ratio = 0.75f;
  p->use_differential = 1;
  p->min_diff_rot = 0.001f;
  p->min_diff_trans = 0.01f;
  p->smooth_length = 4;
  p->cell_size = 0.f;
  p->leaf_split = 0;
  p->max_cells = 0;
  p->reading_sampling_prob = 1.0f;
  p->reference_normals_knn = 0;
  p->reference_sampling_ratio = 1.0f;
  p->unapplied_modules = 0;
}

int ls_check_rigid(const float T[16]) { return check_rigid(T); }
void ls_correct_rigid(const float T_in[16], float T_out[16]) { correct_rigid(T_in, T_out); }

int ls_icp_register(ls_ctx* ctx, const ls_icp_params* prm, const float* reading4, int n, const float* ref4,
                    const float* ref_normals, int normals_stride, int m, const float T0[16], float T_out[16],
                    ls_icp_stats* stats, int32_t* opt_ids, float* opt_d2, float* opt_T_iter_hist) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!reading4 || !ref4 || !ref_normals || !T0 || !T_out || n < 0 || m < 0 || normals_stride < 3)
    return fail(ctx, LS_ERR_ARG, "bad argument");
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  std::memcpy(T_out, T0, 16 * sizeof(float));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  if (n == 0 || m == 0) return fail(ctx, LS_ERR_CONVERGENCE, "empty reading or reference");
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  const Resolved r = resolve(prm);
  if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
  if ((rc = ensure_staging(ctx, n, m))) return rc;
  CU(cudaEventRecord(w->ev0, w->stream));
  CU(cudaMemcpyAsync(ctx->reading, reading4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->ref_stage, ref4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if ((rc = upload_normals(ctx, w, ref_normals, normals_stride, m, ctx->ref_nrm_stage))) return rc;
  Parts parts;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = 1;
  parts.offset[0] = 0;
  parts.offset[1] = m;
  parts.pts[0] = ctx->ref_stage;
  parts.nrm[0] = ctx->ref_nrm_stage;
  parts.identity[0] = 1;
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  return run_icp(ctx, prm, ctx->reading, n, T0, T_out, stats, opt_ids, opt_d2, opt_T_iter_hist);
}

int ls_nn_query(ls_ctx* ctx, const ls_icp_params* prm, const float* reading4, int n, const float* ref4, int m,
                const float T0[16], int32_t* ids, float* d2) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!reading4 || !ref4 || !T0 || !ids || !d2 || n < 0 || m < 0) return fail(ctx, LS_ERR_ARG, "bad argument");
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  if (n == 0) return LS_OK;
  if (m == 0) {
    for (int i = 0; i < n; ++i) { ids[i] = -1; d2[i] = INFINITY; }
    return LS_OK;
  }
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  const Resolved r = resolve(prm);
  if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, 1))) return rc;
  if ((rc = ensure_staging(ctx, n, m))) return rc;
  CU(cudaMemcpyAsync(ctx->reading, reading4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->ref_stage, ref4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemsetAsync(ctx->ref_nrm_stage, 0, (size_t)m * sizeof(float4), w->stream));
  Parts parts;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = 1;
  parts.offset[1] = m;
  parts.pts[0] = ctx->ref_stage;
  parts.nrm[0] = ctx->ref_nrm_stage;
  parts.identity[0] = 1;
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  w->job_host->reading = ctx->reading;
  w->job_host->n = n;
  CU(cudaMemcpyAsync(w->job_dev, w->job_host, sizeof(BuildJob), cudaMemcpyHostToDevice, w->stream));
  reading_kernel<<<dim3(blocks_for(n, 256, ctx->sm_count * 8), 1), 256, 0, w->stream>>>(w->job_dev);
  LAUNCH_CHECK();
  GridView v{w->A.top, w->A.tab1, w->A.srt_pts, w->A.pyr, w->A.topmask};
  nn_query_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->bs, v, w->rd, n, w->ids, w->d2);
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(ids, w->ids, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, w->stream));
  CU(cudaMemcpyAsync(d2, w->d2, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  CU(cudaStreamSynchronize(w->stream));
  return LS_OK;
}

int ls_transform_cloud(ls_ctx* ctx, const float T[16], const float* in4, const float* normals, int normals_stride,
                       int n, float* out4, float* out_normals3) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!T || !in4 || !out4 || n < 0 || (normals && normals_stride < 3) || (normals && !out_normals3))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n == 0) return LS_OK;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  int rc;
  if ((rc = ensure_capacity(ctx, w, n, n, 64, 1))) return rc;
  if ((rc = ensure_staging(ctx, n, n))) return rc;
  CU(cudaMemcpyAsync(ctx->T0_dev, T, 16 * sizeof(float), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->reading, in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if (normals && (rc = upload_normals(ctx, w, normals, normals_stride, n, ctx->ref_nrm_stage))) return rc;
  transform_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(
      ctx->T0_dev, ctx->reading, normals ? ctx->ref_nrm_stage : nullptr, n, w->rd, w->A.sub_nrm);
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(out4, w->rd, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
  if (normals) {
    pack_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->A.sub_nrm, n,
                                                                                         (float*)w->A.srt_nrm);
    LAUNCH_CHECK();
    CU(cudaMemcpyAsync(out_normals3, w->A.srt_nrm, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  }
  CU(cudaStreamSynchronize(w->stream));
  return LS_OK;
}

// ---- rolling map ------------------------------------------------------------------------------------
int ls_map_create(ls_ctx* ctx, int capacity_scans, int max_pts_per_scan, ls_map** out) {
  if (!ctx || !out) return LS_ERR_ARG;
  *out = nullptr;
  if (capacity_scans < 2 || capacity_scans > 4096 || max_pts_per_scan < 1)
    return fail(ctx, LS_ERR_ARG, "bad map geometry");
  CU(cudaSetDevice(ctx->device));
  ls_map* map = new ls_map();
  map->ctx = ctx;
  map->capacity = capacity_scans;
  map->max_pts = max_pts_per_scan;
  map->slots.resize(capacity_scans);
  if (cudaStreamCreateWithFlags(&map->up_stream, cudaStreamNonBlocking) != cudaSuccess) {
    ls_map_destroy(map);
    return fail(ctx, LS_ERR_CUDA, "stream creation failed");
  }
  for (auto& s : map->slots) {
    if (cudaMalloc((void**)&s.pts, (size_t)max_pts_per_scan * sizeof(float4)) != cudaSuccess ||
        cudaMalloc((void**)&s.nrm, (size_t)max_pts_per_scan * sizeof(float4)) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.ready, cudaEventDisableTiming) != cudaSuccess) {
      ls_map_destroy(map);
      return fail(ctx, LS_ERR_NOMEM, "map allocation failed");
    }
  }
  *out = map;
  return LS_OK;
}

void ls_map_destroy(ls_map* map) {
  if (!map) return;
  if (map->ctx) {
    cudaSetDevice(map->ctx->device);
    for (Workspace* w : map->ctx->ws) cudaStreamSynchronize(w->stream);
  }
  if (map->up_stream) cudaStreamSynchronize(map->up_stream);
  for (auto& s : map->slots) {
    if (s.pts) cudaFree(s.pts);
    if (s.nrm) cudaFree(s.nrm);
    if (s.ready) cudaEventDestroy(s.ready);
  }
  for (int k = 0; k < kStageRing; ++k) {
    if (map->host_stage[k]) cudaFreeHost(map->host_stage[k]);
    if (map->stage[k]) cudaFree(map->stage[k]);
    if (map->stage_free[k]) cudaEventDestroy(map->stage_free[k]);
  }
  if (map->up_stream) cudaStreamDestroy(map->up_stream);
  delete map;
}

// The caller's buffers (pageable in general: Eigen / std::vector storage of a DataPoints) are only valid during the
// call, so they are copied into pinned staging memory owned by the map; the transfer to the device then runs on the
// map's upload stream BEHIND the call, and consumers order themselves after it with the slot's event -- exactly the
// asynchronous path, minus the caller's obligation to keep (and pin) its buffers.
int ls_map_push_scan(ls_map* map, const float* features4, const float* normals, int normals_stride, int n,
                     uint64_t* scan_id) {
  if (!map) return LS_ERR_ARG;
  ls_ctx* ctx = map->ctx;
  BUSY_CHECK(ctx);
  if (!features4 || !normals || normals_stride < 3 || n < 0 || n > map->max_pts || !scan_id)
    return fail(ctx, LS_ERR_ARG, "bad argument (n=%d, max=%d)", n, map->max_pts);
  CU(cudaSetDevice(ctx->device));
  if (n == 0) return ls_map_push_scan_async(map, features4, normals, normals_stride > 8 ? 3 : normals_stride, 0, scan_id);
  const int k = (int)(map->n_async % kStageRing);  // the slot of the staging rings the asynchronous push below will take
  if (map->stage_free[k]) CU(cudaEventSynchronize(map->stage_free[k]));  // the upload that used this staging slot last
  const int stride = normals_stride <= 8 ? normals_stride : 3;
  const size_t nf = (size_t)n * 4, nn = (size_t)(n - 1) * (size_t)stride + 3;
  if (nf + nn > map->host_stage_cap[k]) {
    if (map->host_stage[k]) CU(cudaFreeHost(map->host_stage[k]));
    map->host_stage[k] = nullptr;
    map->host_stage_cap[k] = 0;
    if (cudaMallocHost((void**)&map->host_stage[k], (nf + nn + 1024) * sizeof(float)) != cudaSuccess)
      return fail(ctx, LS_ERR_NOMEM, "pinned staging allocation failed");
    map->host_stage_cap[k] = nf + nn + 1024;
  }
  float* hf = map->host_stage[k];
  float* hn = hf + nf;
  std::memcpy(hf, features4, nf * sizeof(float));
  if (normals_stride <= 8) {
    std::memcpy(hn, normals, nn * sizeof(float));  // never past the last normal (the block may start at a row offset)
  } else {
    for (int i = 0; i < n; ++i) {
      const float* r = normals + (size_t)i * (size_t)normals_stride;
      hn[3 * (size_t)i] = r[0]; hn[3 * (size_t)i + 1] = r[1]; hn[3 * (size_t)i + 2] = r[2];
    }
  }
  return ls_map_push_scan_async(map, hf, hn, stride, n, scan_id);
}

// Asynchronous variant: everything is enqueued on the map's own upload stream and the call returns; the host buffers
// must stay valid (and should be pinned, or the copies degrade to synchronous ones) until ls_map_sync or until a
// registration that uses the scan has returned.  Consumers order themselves behind the upload with the slot's event,
// so scan s+1 can go up while scan s is being registered.
int ls_map_push_scan_async(ls_map* map, const float* features4, const float* normals, int normals_stride, int n,
                           uint64_t* scan_id) {
  if (!map) return LS_ERR_ARG;
  ls_ctx* ctx = map->ctx;
  if (!features4 || !normals || normals_stride < 3 || normals_stride > 8 || n < 0 || n > map->max_pts || !scan_id)
    return fail(ctx, LS_ERR_ARG, "bad argument (n=%d, max=%d, 3 <= normals_stride <= 8)", n, map->max_pts);
  CU(cudaSetDevice(ctx->device));
  // The slot this upload evicts must not be one the batch in flight (between _batch_begin and _batch_end) still reads:
  // its assemble / reading kernels run on other streams and are not ordered against this copy.  Every other consumer
  // of a slot is a synchronous call, so it has returned; uploads into the same slot are ordered by the upload stream.
  const int slot_index = (int)(map->next_id % (uint64_t)map->capacity);
  if (ctx->pending)
    for (const auto& ps : ctx->pending_slots)
      if (ps.first == map && ps.second == slot_index)
        return fail(ctx, LS_ERR_STATE, "ring slot %d is read by the batch in flight (capacity %d too small for the scans in flight)",
                    slot_index, map->capacity);
  const uint64_t id = map->next_id++;
  ls_scan_slot& s = map->slots[id % (uint64_t)map->capacity];
  s.used = false;
  if (n > 0) {
    const int k = (int)(map->n_async++ % kStageRing);
    const size_t need = (size_t)(n - 1) * (size_t)normals_stride + 3;  // never read past the last normal
    if (!map->stage_free[k]) CU(cudaEventCreateWithFlags(&map->stage_free[k], cudaEventDisableTiming));
    else CU(cudaEventSynchronize(map->stage_free[k]));  // the upload that used this staging buffer 16 pushes ago
    if (need > map->stage_cap[k]) {
      if (map->stage[k]) CU(cudaFree(map->stage[k]));
      map->stage[k] = nullptr;
      map->stage_cap[k] = 0;
      if (cudaMalloc((void**)&map->stage[k], (need + 1024) * sizeof(float)) != cudaSuccess)
        return fail(ctx, LS_ERR_NOMEM, "staging allocation failed");
      map->stage_cap[k] = need + 1024;
    }
    CU(cudaMemcpyAsync(s.pts, features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, map->up_stream));
    CU(cudaMemcpyAsync(map->stage[k], normals, need * sizeof(float), cudaMemcpyHostToDevice, map->up_stream));
    expand_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, map->up_stream>>>(map->stage[k], normals_stride, n, s.nrm);
    LAUNCH_CHECK();
    CU(cudaEventRecord(map->stage_free[k], map->up_stream));
  }
  CU(cudaEventRecord(s.ready, map->up_stream));
  s.async = true;
  s.n = n;
  s.id = id;
  s.used = true;
  *scan_id = id;
  return LS_OK;
}

int ls_host_is_pinned(const void* p) {
  if (!p) return LS_ERR_ARG;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return a.type == cudaMemoryTypeHost ? 1 : 0;
}

int ls_map_sync(ls_map* map) {
  if (!map) return LS_ERR_ARG;
  ls_ctx* ctx = map->ctx;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(map->up_stream));
  return LS_OK;
}

namespace {
// Normals of a device-resident cloud (float4, scan frame) into nrm_out (float4, same order): build the cloud's own
// spatial hash on workspace 0, then exact kNN + covariance + smallest eigenvector per point.
int enqueue_normals(ls_ctx* ctx, Workspace* w, const float4* pts_dev, int n, int knn, float4* nrm_out) {
  ls_icp_params dflt;
  ls_icp_default_params(&dflt);
  const Resolved r = resolve(&dflt);
  int rc;
  if ((rc = ensure_capacity(ctx, w, n, n, r.max_cells, 1))) return rc;
  Parts parts;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = 1;
  parts.offset[1] = n;
  parts.pts[0] = pts_dev;
  parts.nrm[0] = pts_dev;  // normals are an output here; the assembly pass just needs a readable array
  parts.identity[0] = 1;
  const float I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if ((rc = enqueue_build(ctx, w, parts, r, I))) return rc;
  GridView v{w->A.top, w->A.tab1, w->A.srt_pts, w->A.pyr, w->A.topmask};
  knn_normals_kernel<<<blocks_for(n, 128, ctx->sm_count * 16), 128, 0, w->stream>>>(w->bs, v, w->A.sub_pts, n, knn, nrm_out);
  LAUNCH_CHECK();
  return LS_OK;
}
}  // namespace

int ls_estimate_normals(ls_ctx* ctx, const float* features4, int n, int knn, float* out_normals3) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!features4 || !out_normals3 || n < 0 || knn < 3 || knn > LS_KNN_MAX) return fail(ctx, LS_ERR_ARG, "bad argument (3 <= knn <= %d)", LS_KNN_MAX);
  if (n == 0) return LS_OK;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  int rc;
  if ((rc = ensure_capacity(ctx, w, n, n, 64, 1))) return rc;
  if ((rc = ensure_staging(ctx, n, n))) return rc;
  CU(cudaMemcpyAsync(ctx->reading, features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if ((rc = enqueue_normals(ctx, w, ctx->reading, n, knn, ctx->ref_nrm_stage))) return rc;
  pack_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(ctx->ref_nrm_stage, n, (float*)w->A.srt_nrm);
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(out_normals3, w->A.srt_nrm, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  CU(cudaStreamSynchronize(w->stream));
  return LS_OK;
}

int ls_map_push_scan_estimate_normals(ls_map* map, const float* features4, int n, int knn, uint64_t* scan_id) {
  if (!map) return LS_ERR_ARG;
  ls_ctx* ctx = map->ctx;
  BUSY_CHECK(ctx);
  if (!features4 || n < 0 || n > map->max_pts || !scan_id || knn < 3 || knn > LS_KNN_MAX)
    return fail(ctx, LS_ERR_ARG, "bad argument (n=%d, max=%d, 3 <= knn <= %d)", n, map->max_pts, LS_KNN_MAX);
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  const uint64_t id = map->next_id++;
  ls_scan_slot& s = map->slots[id % (uint64_t)map->capacity];
  s.used = false;
  if (s.async) {
    CU(cudaEventSynchronize(s.ready));
    s.async = false;
  }
  if (n > 0) {
    CU(cudaMemcpyAsync(s.pts, features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
    int rc = enqueue_normals(ctx, w, s.pts, n, knn, s.nrm);
    if (rc) return rc;
    CU(cudaStreamSynchronize(w->stream));
  }
  s.n = n;
  s.id = id;
  s.used = true;
  *scan_id = id;
  return LS_OK;
}

int ls_map_scan_size(const ls_map* map, uint64_t scan_id) {
  if (!map) return LS_ERR_ARG;
  const ls_scan_slot* s = find_slot(map, scan_id);
  return s ? s->n : LS_ERR_STATE;
}

int ls_icp_register_submap(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, uint64_t reading_id, int n_parts,
                           const uint64_t* part_ids, const float* T_parts, const float T0[16], float T_out[16],
                           ls_icp_stats* stats, int32_t* opt_ids, float* opt_d2, float* opt_T_iter_hist) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!map || map->ctx != ctx || !part_ids || !T_parts || !T0 || !T_out) return fail(ctx, LS_ERR_ARG, "bad argument");
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  std::memcpy(T_out, T0, 16 * sizeof(float));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  const ls_scan_slot* rs = find_slot(map, reading_id);
  if (!rs) return fail(ctx, LS_ERR_STATE, "reading scan %llu is not resident", (unsigned long long)reading_id);
  Parts parts;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  if ((rc = make_parts(ctx, map, n_parts, part_ids, T_parts, &parts, w->stream))) return rc;
  if (wait_slot(rs, w->stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
  const int n = rs->n, m = parts.offset[n_parts];
  if (n == 0 || m == 0) return fail(ctx, LS_ERR_CONVERGENCE, "empty reading or reference");
  const Resolved r = resolve(prm);
  if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
  CU(cudaEventRecord(w->ev0, w->stream));
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  return run_icp(ctx, prm, rs->pts, n, T0, T_out, stats, opt_ids, opt_d2, opt_T_iter_hist);
}

// ---- query-sharded registration (SURVEY.md 8 e-2) -------------------------------------------------------------
// ONE registration whose reading is split over the GPUs of a node.  Every shard holds the whole map (the build is
// replicated: it costs ~54 us) and a contiguous range of the cell-sorted reading.  Per iteration the shards exchange
// their partial select histograms and their 28 partial normal-equation sums: each GPU pushes its sections into a slot
// of every peer's exchange buffer (peer-mapped with CUDA IPC, plain stores over NVLink) from inside the persistent
// kernel and bumps the peer's arrival counter; readers sum the slots, all local (ShardLink, shard_exchange in
// ls_kernels.cuh).  No collective call, no host involvement per iteration, nothing polled across NVLink.  All the sums
// are integers, so the result is bit-identical to the unsharded registration whatever the number of shards.
namespace {
size_t xbuf_bytes(int shards) { return sizeof(IcpWork) * (size_t)shards + 128; }
}

int ls_shard_exchange_create(ls_ctx* ctx, int shard_rank, int shard_count, unsigned char handle[LS_IPC_HANDLE_BYTES]) {
  if (!ctx || !handle) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  static_assert(sizeof(cudaIpcMemHandle_t) <= LS_IPC_HANDLE_BYTES, "handle size");
  if (shard_count < 1 || shard_count > kMaxShards || shard_rank < 0 || shard_rank >= shard_count)
    return fail(ctx, LS_ERR_ARG, "shard %d of %d (at most %d shards)", shard_rank, shard_count, kMaxShards);
  CU(cudaSetDevice(ctx->device));
  ls_shard_exchange_close(ctx);
  CU(cudaMalloc((void**)&ctx->xbuf, xbuf_bytes(shard_count)));
  CU(cudaMemset(ctx->xbuf, 0, xbuf_bytes(shard_count)));
  CU(cudaDeviceSynchronize());
  ctx->shard_rank = shard_rank;
  ctx->shard_count = shard_count;
  ctx->xflag_base = 0;
  ctx->xconnected = shard_count == 1;
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, ctx->xbuf));
  std::memset(handle, 0, LS_IPC_HANDLE_BYTES);
  std::memcpy(handle, &h, sizeof(h));
  return LS_OK;
}

int ls_shard_exchange_connect(ls_ctx* ctx, const unsigned char* handles) {
  if (!ctx || !handles) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!ctx->xbuf) return fail(ctx, LS_ERR_STATE, "ls_shard_exchange_create first");
  CU(cudaSetDevice(ctx->device));
  for (int g = 0; g < ctx->shard_count; ++g) {
    if (g == ctx->shard_rank || ctx->xpeer[g]) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handles + (size_t)g * LS_IPC_HANDLE_BYTES, sizeof(h));
    void* p = nullptr;
    CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->xpeer[g] = static_cast<unsigned char*>(p);
  }
  ctx->xconnected = true;
  return LS_OK;
}

void ls_shard_exchange_close(ls_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (int g = 0; g < kMaxShards; ++g) {
    if (ctx->xpeer[g]) cudaIpcCloseMemHandle(ctx->xpeer[g]);
    ctx->xpeer[g] = nullptr;
  }
  if (ctx->xbuf) cudaFree(ctx->xbuf);
  ctx->xbuf = nullptr;
  ctx->xconnected = false;
  ctx->shard_count = 1;
  ctx->shard_rank = 0;
}

int ls_icp_register_submap_sharded(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, uint64_t reading_id, int n_parts,
                                   const uint64_t* part_ids, const float* T_parts, const float T0[16], float T_out[16],
                                   ls_icp_stats* stats) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!map || map->ctx != ctx || !part_ids || !T_parts || !T0 || !T_out) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!ctx->xbuf || !ctx->xconnected)
    return fail(ctx, LS_ERR_STATE, "no exchange buffer: ls_shard_exchange_create + ls_shard_exchange_connect first");
  const int shard_rank = ctx->shard_rank, shard_count = ctx->shard_count;
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  std::memcpy(T_out, T0, 16 * sizeof(float));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  const ls_scan_slot* rs = find_slot(map, reading_id);
  if (!rs) return fail(ctx, LS_ERR_STATE, "reading scan %llu is not resident", (unsigned long long)reading_id);
  Parts parts;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  if ((rc = make_parts(ctx, map, n_parts, part_ids, T_parts, &parts, w->stream))) return rc;
  if (wait_slot(rs, w->stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
  const int n = rs->n, m = parts.offset[n_parts];
  if (n == 0 || m == 0) return fail(ctx, LS_ERR_CONVERGENCE, "empty reading or reference");
  const Resolved r = resolve(prm);
  if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
  CU(cudaEventRecord(w->ev0, w->stream));
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  if ((rc = prep_icp(ctx, w, prm, rs->pts, n, T0, false, false))) return rc;
  IcpProblem& hp = w->hp;
  hp.shard_rank = shard_rank;
  hp.shard_count = shard_count;
  if (shard_count > 1) {
    IcpWork* slots = reinterpret_cast<IcpWork*>(ctx->xbuf);
    // this shard's own slot starts from zero; the peers' slots are overwritten section by section before they are read
    CU(cudaMemsetAsync(slots + shard_rank, 0, sizeof(IcpWork), w->stream));
    hp.link.slots = slots;
    hp.link.flag = reinterpret_cast<unsigned int*>(ctx->xbuf + sizeof(IcpWork) * (size_t)shard_count);
    hp.link.flag_base = ctx->xflag_base;
    for (int g = 0; g < kMaxShards; ++g) {
      unsigned char* pb = g < shard_count ? ctx->xpeer[g] : nullptr;
      hp.link.peer_slots[g] = reinterpret_cast<IcpWork*>(pb);
      hp.link.peer_flag[g] = pb ? reinterpret_cast<unsigned int*>(pb + sizeof(IcpWork) * (size_t)shard_count) : nullptr;
    }
  }
  // every shard runs the full co-resident grid (the exchange needs a CTA per peer, and all shards the same shape)
  if ((rc = launch_icp(ctx, prm, 1, 1 << 30, shard_count > 1))) return rc;
  CU(cudaStreamSynchronize(w->stream));
  ctx->xflag_base += w->h_work->xsignals;
  return fetch_icp(ctx, w, n, T0, T_out, stats);
}

// Sub-map <-> sub-map registration with both clouds assembled on the device (SURVEY.md 8 f2: the loop-closure ICP of
// IncrementalEstimator::processLoopClosure, reference incremental_estimator.cpp:90-115, whose two
// buildSubMapAroundTime clouds never have to visit the host).  Bit-identical to ls_map_assemble of both sides
// followed by ls_icp_register.
int ls_icp_register_submaps(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* ref_map, int n_ref_parts,
                            const uint64_t* ref_part_ids, const float* T_ref_parts, const ls_map* reading_map,
                            int n_reading_parts, const uint64_t* reading_part_ids, const float* T_reading_parts,
                            const float T0[16], float T_out[16], ls_icp_stats* stats) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!ref_map || ref_map->ctx != ctx || !reading_map || reading_map->ctx != ctx || !ref_part_ids || !T_ref_parts ||
      !reading_part_ids || !T_reading_parts || !T0 || !T_out)
    return fail(ctx, LS_ERR_ARG, "bad argument");
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  std::memcpy(T_out, T0, 16 * sizeof(float));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  Parts ref, rd;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  if ((rc = make_parts(ctx, ref_map, n_ref_parts, ref_part_ids, T_ref_parts, &ref, w->stream))) return rc;
  if ((rc = make_parts(ctx, reading_map, n_reading_parts, reading_part_ids, T_reading_parts, &rd, w->stream))) return rc;
  const int n = rd.offset[n_reading_parts], m = ref.offset[n_ref_parts];
  if (n == 0 || m == 0) return fail(ctx, LS_ERR_CONVERGENCE, "empty reading or reference");
  const Resolved r = resolve(prm);
  if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
  if ((rc = ensure_staging(ctx, n, 0))) return rc;
  CU(cudaEventRecord(w->ev0, w->stream));
  assemble_points_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(rd, ctx->reading);
  LAUNCH_CHECK();
  if ((rc = enqueue_build(ctx, w, ref, r, T0))) return rc;
  return run_icp(ctx, prm, ctx->reading, n, T0, T_out, stats, nullptr, nullptr, nullptr);
}

// Several independent scan -> sub-map registrations in ONE cooperative launch (the multi-robot case: the
// reference's n_laser_slam_workers tracks, reference incremental_estimator.cpp:22-26, hosted on one GPU).
// Problem b stages on its own stream (assembly + hash build overlap across problems); the persistent kernel's
// grid is split into `batch` CTA groups, each with its own barrier, so one problem's barrier / solve latency is
// filled by the others' search.  Results are bit-identical to `batch` separate ls_icp_register_submap calls.
int ls_icp_register_submap_batch_begin(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, int batch,
                                       const uint64_t* reading_ids, const int* n_parts, const uint64_t* part_ids,
                                       const float* T_parts, const float* T0s) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!map || map->ctx != ctx || batch < 1 || batch > kMaxBatch || !reading_ids || !n_parts || !part_ids || !T_parts || !T0s)
    return fail(ctx, LS_ERR_ARG, "bad argument (1 <= batch <= %d)", kMaxBatch);
  int rc = check_params(ctx, prm);
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  if ((rc = ensure_workspaces(ctx, batch))) return rc;
  const Resolved r = resolve(prm);
  ctx->pending_n.assign(batch, 0);
  ctx->pending_T0.assign(T0s, T0s + 16 * (size_t)batch);
  ctx->pending_slots.clear();
  // validate every problem before anything is enqueued
  {
    int po = 0;
    for (int b = 0; b < batch; ++b) {
      if (n_parts[b] < 1 || n_parts[b] > kMaxParts) return fail(ctx, LS_ERR_ARG, "n_parts must be in [1,%d]", kMaxParts);
      const ls_scan_slot* rs = find_slot(map, reading_ids[b]);
      if (!rs) return fail(ctx, LS_ERR_STATE, "reading scan %llu is not resident", (unsigned long long)reading_ids[b]);
      if (rs->n == 0) return fail(ctx, LS_ERR_ARG, "empty reading in a batch (use the single call)");
      ctx->pending_slots.emplace_back(map, (int)(rs - map->slots.data()));
      long long m = 0;
      for (int p = 0; p < n_parts[b]; ++p) {
        const ls_scan_slot* s = find_slot(map, part_ids[po + p]);
        if (!s) return fail(ctx, LS_ERR_STATE, "scan %llu is not resident (evicted or never pushed)", (unsigned long long)part_ids[po + p]);
        ctx->pending_slots.emplace_back(map, (int)(s - map->slots.data()));
        m += s->n;
      }
      if (m == 0) return fail(ctx, LS_ERR_ARG, "empty reference in a batch (use the single call)");
      po += n_parts[b];
    }
  }
  // stage every problem's job on the host, then ONE upload and ONE launch per build phase for the whole batch
  Workspace* w0 = ctx->ws[0];
  int n_max = 0, m_max = 0, part_off = 0;
  for (int b = 0; b < batch; ++b) {
    Workspace* w = ctx->ws[b];
    const float* T0 = T0s + 16 * b;
    const ls_scan_slot* rs = find_slot(map, reading_ids[b]);
    Parts parts;
    if ((rc = make_parts(ctx, map, n_parts[b], part_ids + part_off, T_parts + 16 * (size_t)part_off, &parts, w0->stream)))
      return rc;
    if (wait_slot(rs, w0->stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
    part_off += n_parts[b];
    const int n = rs->n, m = parts.offset[n_parts[b]];
    ctx->pending_n[b] = n;
    n_max = n > n_max ? n : n_max;
    m_max = m > m_max ? m : m_max;
    if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
    fill_job(w, parts, T0, rs->pts, n);
    if ((rc = fill_problem(ctx, w, prm, n, T0, false, false))) return rc;
  }
  for (int b = 1; b < batch; ++b) {  // allocation-time clears a workspace enqueued on its own stream come first
    if (!ctx->ws[b]->stream_dirty) continue;
    CU(cudaEventRecord(ctx->ws[b]->ev2, ctx->ws[b]->stream));
    CU(cudaStreamWaitEvent(w0->stream, ctx->ws[b]->ev2, 0));
    ctx->ws[b]->stream_dirty = false;
  }
  CU(cudaEventRecord(w0->ev0, w0->stream));
  CU(cudaMemcpyAsync(ctx->jobs_dev, ctx->jobs_host, sizeof(BuildJob) * (size_t)batch, cudaMemcpyHostToDevice, w0->stream));
  if ((rc = launch_build(ctx, ctx->jobs_dev, batch, m_max, r, w0->stream))) return rc;
  if ((rc = launch_reading_sort(ctx, ctx->jobs_dev, batch, n_max, r, w0->stream))) return rc;
  CU(cudaEventRecord(w0->ev1, w0->stream));
  CU(cudaMemsetAsync(ctx->work_pool, 0, sizeof(IcpWork) * (size_t)batch, w0->stream));
  if ((rc = launch_icp(ctx, prm, batch, n_max))) return rc;
  ctx->pending_batch = batch;
  ctx->pending = true;
  return LS_OK;
}

int ls_icp_register_submap_batch_end(ls_ctx* ctx, float* T_outs, ls_icp_stats* stats, int* statuses) {
  if (!ctx) return LS_ERR_ARG;
  if (!ctx->pending) return fail(ctx, LS_ERR_STATE, "no batch in flight");
  if (!T_outs || !statuses) return fail(ctx, LS_ERR_ARG, "bad argument");
  ctx->pending = false;
  ctx->pending_slots.clear();
  const int batch = ctx->pending_batch;
  std::memcpy(T_outs, ctx->pending_T0.data(), 16 * sizeof(float) * (size_t)batch);
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->ws[0]->stream));
  for (int b = 0; b < batch; ++b) {
    const int st = fetch_icp(ctx, ctx->ws[b], ctx->pending_n[b], ctx->pending_T0.data() + 16 * b, T_outs + 16 * b,
                             stats ? stats + b : nullptr, true);
    if (st < 0) return st;
    statuses[b] = st;
  }
  return LS_OK;
}

int ls_icp_register_submap_batch(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, int batch,
                                 const uint64_t* reading_ids, const int* n_parts, const uint64_t* part_ids,
                                 const float* T_parts, const float* T0s, float* T_outs, ls_icp_stats* stats, int* statuses) {
  if (!ctx) return LS_ERR_ARG;
  if (!T_outs || !statuses) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (T0s && batch >= 1 && batch <= kMaxBatch) std::memcpy(T_outs, T0s, 16 * sizeof(float) * (size_t)batch);
  const int rc = ls_icp_register_submap_batch_begin(ctx, prm, map, batch, reading_ids, n_parts, part_ids, T_parts, T0s);
  if (rc != LS_OK) return rc;
  return ls_icp_register_submap_batch_end(ctx, T_outs, stats, statuses);
}

int ls_map_assemble(ls_ctx* ctx, const ls_map* map, int n_parts, const uint64_t* part_ids, const float* T_parts,
                    float* out4, float* out_normals3, int* m_out) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!map || map->ctx != ctx || !part_ids || !T_parts || !out4 || !m_out) return fail(ctx, LS_ERR_ARG, "bad argument");
  Parts parts;
  int rc;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  if ((rc = make_parts(ctx, map, n_parts, part_ids, T_parts, &parts, w->stream))) return rc;
  const int m = parts.offset[n_parts];
  *m_out = m;
  if (m == 0) return LS_OK;
  if ((rc = ensure_capacity(ctx, w, 1, m, 64, 1))) return rc;
  const float I16[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  fill_job(w, parts, I16, nullptr, 0);
  CU(cudaMemcpyAsync(w->job_dev, w->job_host, sizeof(BuildJob), cudaMemcpyHostToDevice, w->stream));
  reset_build_kernel<<<dim3(1, 1), 32, 0, w->stream>>>(w->job_dev);
  LAUNCH_CHECK();
  assemble_kernel<<<dim3(blocks_for(m, 256, ctx->sm_count * 8), 1), 256, 0, w->stream>>>(w->job_dev);
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(out4, w->A.sub_pts, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
  if (out_normals3) {
    pack_normals_kernel<<<blocks_for(m, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->A.sub_nrm, m,
                                                                                         (float*)w->A.srt_nrm);
    LAUNCH_CHECK();
    CU(cudaMemcpyAsync(out_normals3, w->A.srt_nrm, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  }
  CU(cudaStreamSynchronize(w->stream));
  return LS_OK;
}

}  // extern "C"
