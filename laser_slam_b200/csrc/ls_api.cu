// C-ABI implementation (include/ls_b200.h): context, device memory, kernel launches.
// There is no CPU fallback anywhere in this file: every entry point needs a live CUDA device.
#include <cerrno>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ls_b200.h"
#include "ls_buffer.cuh"
#include "ls_filters.cuh"
#include "ls_kernels.cuh"
#include "ls_occupancy.cuh"

using namespace ls;

#define LS_VERSION 100

// Everything one registration needs on the device.  A context owns one workspace per concurrently
// running problem (ls_icp_register_submap_batch); single-problem entry points use workspace 0.
// The arrays come in groups that grow together (ensure_capacity); the first array of a group tells its capacity.
struct Workspace {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev_launch = nullptr;
  Buffer<BuildState> bs;
  // per reading point
  Buffer<float4> rd;  // pre-transformed reading
  Buffer<int> pos;
  Buffer<float> d2;
  Buffer<float4> vq, vpts;  // certified candidate lists (ls_grid.cuh VLists)
  Buffer<int> ids;
  Buffer<float> d2_out;
  Buffer<uint32_t> qkey, qperm;
  Buffer<float4> rd_s;
  // per sub-map point, and the fine tables (BuildArrays)
  Buffer<float4> sub_pts, sub_nrm, srt_pts, srt_nrm;
  Buffer<uint32_t> pkey;
  Buffer<Entry> tab1;
  Buffer<uint32_t> cnt1, tab1_cell, qtab_local, qtab_total;
  // per level-0 cell
  Buffer<Entry> top;
  Buffer<uint32_t> cnt0;
  Buffer<unsigned long long> pyr, topmask;
  Buffer<uint32_t> qtop_start;
  Buffer<float> T_hist;  // per iteration
  IcpWork* work = nullptr;
  BuildJob* job_host = nullptr;  // pinned; this workspace's slot of the context's job array
  BuildJob* job_dev = nullptr;
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
  Buffer<IcpProblem> probs_dev;          // [kMaxBatch]
  PinnedBuffer<IcpProblem> probs_host;
  Buffer<BuildJob> jobs_dev;             // [kMaxBatch]: workspace b stages its build in slot b
  PinnedBuffer<BuildJob> jobs_host;
  Buffer<IcpWork> work_pool;             // [kMaxBatch] contiguous, so one memset clears a whole batch
  Buffer<IcpResult> results_dev;         // [kMaxBatch]: launch_icp gathers every problem's results here ...
  PinnedBuffer<IcpResult> results_host;  // ... and copies them back in one piece
  // staging of the entry points that take host clouds (used on workspace 0's stream; ensure_staging)
  Buffer<float4> reading;                 // raw reading
  Buffer<float4> ref_stage, ref_nrm_stage;  // reference points and normals (scan frame)
  Buffer<float> nrm_raw;                  // raw normals (upload_normals)
  Buffer<float> T0_dev;                   // 16 floats: ls_transform_cloud's transformation
  // query-sharded registration: this GPU's exchange buffer (shard_count slots + the arrival counter) and the peers'
  unsigned char* xbuf = nullptr;
  unsigned char* xpeer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int shard_rank = 0, shard_count = 1;
  bool xconnected = false;
  unsigned int xflag_base = 0;  // arrivals the earlier registrations consumed from the counter
  // a batch between ls_icp_register_submap_batch_begin and _end: the workspaces are busy
  bool pending = false;
  int pending_batch = 0;
  std::vector<int> pending_ws;  // per problem of the caller: its workspace, or -1 (empty reading or sub-map: not launched)
  std::vector<int> pending_n;   // per launched problem (workspace order)
  std::vector<float> pending_T0;
  // ring slots (map, slot index) the in-flight batch reads: an asynchronous upload must not overwrite them
  std::vector<std::pair<const ls_map*, int>> pending_slots;
  // device scratch of the per-scan input filters (ls_filter_cloud / ls_map_push_scan_filtered)
  lsf::ChainBuffers chain;
};
constexpr int kMaxBatch = 160;

struct ls_scan_slot {
  Buffer<float4> pts, nrm;
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
  Buffer<float> stage[kStageRing];
  cudaEvent_t stage_free[kStageRing] = {};
  uint64_t n_async = 0;
  // pinned host staging of ls_map_push_scan (pageable caller memory is copied here, the DMA then runs behind the call)
  PinnedBuffer<float> host_stage[kStageRing];
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

// A failed lso:: call (the occupancy map's modules): "<what>: out of device memory" for LS_ERR_NOMEM, else "<what> failed".
int fail_lso(ls_ctx* ctx, int rc, const char* what) {
  return fail(ctx, rc, rc == LS_ERR_NOMEM ? "%s: out of device memory" : "%s failed", what);
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

inline int blocks_for(int n, int threads, int cap) {
  int b = (n + threads - 1) / threads;
  if (b < 1) b = 1;
  return b > cap ? cap : b;
}

// A group of arrays that failed to grow (and was emptied), reported as CU reports a failed call.
int grow_failed(ls_ctx* ctx, cudaError_t e, const char* group) {
  return fail(ctx, e == cudaErrorMemoryAllocation ? LS_ERR_NOMEM : LS_ERR_CUDA, "%s: %s", group, cudaGetErrorString(e));
}

// Each group grows all or nothing: when one array fails, the whole group is emptied, so a later call regrows all of it.
int ensure_capacity(ls_ctx* ctx, Workspace* w, int n, int m, int max_cells, int max_iter) {
  cudaError_t e;
  if ((size_t)n > w->rd.capacity()) {
    const size_t c = (size_t)(n + n / 8 + 1024), cv = c * LS_VK;
    if ((e = w->rd.reserve(c, c)) || (e = w->pos.reserve(c, c)) || (e = w->d2.reserve(c, c)) || (e = w->vq.reserve(c, c)) ||
        (e = w->vpts.reserve(cv, cv)) || (e = w->ids.reserve(c, c)) || (e = w->d2_out.reserve(c, c)) ||
        (e = w->qkey.reserve(c, c)) || (e = w->qperm.reserve(c, c)) || (e = w->rd_s.reserve(c, c))) {
      w->rd.reset(), w->pos.reset(), w->d2.reset(), w->vq.reset(), w->vpts.reset(), w->ids.reset(), w->d2_out.reset();
      w->qkey.reset(), w->qperm.reset(), w->rd_s.reset();
      return grow_failed(ctx, e, "reading arrays");
    }
  }
  if ((size_t)m > w->sub_pts.capacity()) {
    const int cap = m + m / 8 + 1024;
    // a fine table exists only for a level-0 cell with > leaf_split (>= 16) points; the pool is also capped at
    // ~1.5 GB (cells beyond the pool stay leaves: slower, still exact, flagged in stats.grid_overflow)
    int tcap = cap / 17 + 1024;
    const int tmax = (int)((size_t)1536 * 1024 * 1024 / ((size_t)LS_FB3 * 12));
    if (tcap > tmax) tcap = tmax;
    const size_t c = (size_t)cap, t = (size_t)tcap, tf = t * LS_FB3;
    if ((e = w->sub_pts.reserve(c, c)) || (e = w->sub_nrm.reserve(c, c)) || (e = w->srt_pts.reserve(c, c)) ||
        (e = w->srt_nrm.reserve(c, c)) || (e = w->pkey.reserve(c, c)) || (e = w->tab1.reserve(tf, tf)) ||
        (e = w->cnt1.reserve(tf, tf)) || (e = w->tab1_cell.reserve(t, t)) || (e = w->qtab_local.reserve(tf, tf)) ||
        (e = w->qtab_total.reserve(t, t))) {
      w->sub_pts.reset(), w->sub_nrm.reset(), w->srt_pts.reset(), w->srt_nrm.reset(), w->pkey.reset(), w->tab1.reset();
      w->cnt1.reset(), w->tab1_cell.reset(), w->qtab_local.reset(), w->qtab_total.reset();
      return grow_failed(ctx, e, "sub-map arrays");
    }
    CU(cudaMemsetAsync(w->cnt1.get(), 0, tf * sizeof(uint32_t), w->stream));
    w->stream_dirty = true;
  }
  if ((size_t)max_cells + 1 > w->top.capacity()) {
    const size_t c = (size_t)max_cells + 1, cp = (size_t)max_cells / 2 + 4096;
    if ((e = w->top.reserve(c, c)) || (e = w->cnt0.reserve(c, c)) || (e = w->pyr.reserve(cp, cp)) ||
        (e = w->topmask.reserve(c, c)) || (e = w->qtop_start.reserve(c, c))) {
      w->top.reset(), w->cnt0.reset(), w->pyr.reset(), w->topmask.reset(), w->qtop_start.reset();
      return grow_failed(ctx, e, "cell arrays");
    }
    CU(cudaMemsetAsync(w->cnt0.get(), 0, c * sizeof(uint32_t), w->stream));
    w->stream_dirty = true;
  }
  CU(w->T_hist.reserve((size_t)max_iter * 16, (size_t)max_iter * 16));
  return LS_OK;
}

// The kernels' view of workspace w's arrays.
BuildArrays arrays(const Workspace* w) {
  BuildArrays A;
  A.sub_pts = w->sub_pts.get();
  A.sub_nrm = w->sub_nrm.get();
  A.srt_pts = w->srt_pts.get();
  A.srt_nrm = w->srt_nrm.get();
  A.pkey = w->pkey.get();
  A.top = w->top.get();
  A.cnt0 = w->cnt0.get();
  A.tab1 = w->tab1.get();
  A.cnt1 = w->cnt1.get();
  A.tab1_cell = w->tab1_cell.get();
  A.tab_cap = (int)w->tab1_cell.capacity();
  A.pyr = w->pyr.get();
  A.topmask = w->topmask.get();
  A.qkey = w->qkey.get();
  A.qtop_start = w->qtop_start.get();
  A.qtab_local = w->qtab_local.get();
  A.qtab_total = w->qtab_total.get();
  A.qperm = w->qperm.get();
  A.rd_s = w->rd_s.get();
  return A;
}

// The context's staging for a host reading of n points and a host reference of m points, grown like the workspaces.
int ensure_staging(ls_ctx* ctx, int n, int m) {
  const size_t cn = (size_t)(n + n / 8 + 1024), cm = (size_t)(m + m / 8 + 1024);
  CU(ctx->reading.reserve((size_t)n, cn));
  if ((size_t)m > ctx->ref_stage.capacity()) {
    cudaError_t e;
    if ((e = ctx->ref_stage.reserve(cm, cm)) || (e = ctx->ref_nrm_stage.reserve(cm, cm))) {
      ctx->ref_stage.reset(), ctx->ref_nrm_stage.reset();
      return grow_failed(ctx, e, "reference staging");
    }
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
  J.bs = w->bs.get();
  J.A = arrays(w);
  J.m = parts.offset[parts.n_parts];
  J.n = n;
  J.reading = reading_dev;
  J.rd = w->rd.get();
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
  // Many CTAs per job (one point per thread up to 16 CTAs per SM): the CTAs start in job order, more of them than fit on
  // the device at once, so about one job's scatter is in flight at a time and its sorted
  // arrays (32 B per point) stay in L2 until the scattered 16-byte writes have filled their sectors.  Grid-striding
  // every job over 2 CTAs per SM instead keeps several jobs' arrays open at once, more than L2 holds.
  scatter_kernel<<<dim3(blocks_for(m_max, 256, ctx->sm_count * 16), B), 256, 0, st>>>(jobs_dev);
  LAUNCH_CHECK();
  return LS_OK;
}

// R' = T_refMean_dataIn * R for every staged job, and the readings ordered by their map's cell keys (q_count_kernel
// does both in one pass).
int launch_reading_sort(ls_ctx* ctx, const BuildJob* jobs_dev, int batch, int n_max, const Resolved& r, cudaStream_t st) {
  const unsigned int B = (unsigned int)batch;
  const int cap = batch > 1 ? ctx->sm_count * 2 : ctx->sm_count * 8;
  const int qb = blocks_for(n_max, 256, cap);
  const int scan_tiles = (r.max_cells + kScanTile - 1) / kScanTile;
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
  CU(ctx->nrm_raw.reserve(need, need + 4096));
  int dstride = stride;
  if (stride <= 8) {
    CU(cudaMemcpyAsync(ctx->nrm_raw.get(), normals, need * sizeof(float), cudaMemcpyHostToDevice, w->stream));
  } else {
    CU(cudaMemcpy2DAsync(ctx->nrm_raw.get(), 3 * sizeof(float), normals, (size_t)stride * sizeof(float), 3 * sizeof(float),
                         (size_t)n, cudaMemcpyHostToDevice, w->stream));
    dstride = 3;
  }
  expand_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(ctx->nrm_raw.get(), dstride, n, dst);
  LAUNCH_CHECK();
  return LS_OK;
}

// Fill workspace w's problem descriptor for the persistent ICP kernel (host side only).
int fill_problem(ls_ctx* ctx, Workspace* w, const ls_icp_params* prm, int n, const float T0[16], bool want_matches,
                 bool want_hist) {
  IcpProblem& hp = w->hp;
  hp.bs = w->bs.get();
  hp.view.top = w->top.get();
  hp.view.tab1 = w->tab1.get();
  hp.view.pts = w->srt_pts.get();
  hp.view.pyr = w->pyr.get();
  hp.view.topmask = w->topmask.get();
  hp.nrm = w->srt_nrm.get();
  hp.rd = w->rd_s.get();
  hp.n = n;
  hp.pos = w->pos.get();
  hp.d2 = w->d2.get();
  hp.ids = w->ids.get();
  hp.d2_out = w->d2_out.get();
  hp.qperm = w->qperm.get();
  hp.lists.vq = w->vq.get();
  hp.lists.vpts = w->vpts.get();
  hp.lists.n = n;
  hp.work = w->work;
  hp.shard_rank = 0;
  hp.shard_count = 1;
  std::memset(&hp.link, 0, sizeof(hp.link));
  hp.T_hist = want_hist ? w->T_hist.get() : nullptr;
  if (want_hist) {  // entries past the executed iterations read as zeros, not as stale device memory
    CU(cudaMemsetAsync(w->T_hist.get(), 0, (size_t)prm->max_iterations * 16 * sizeof(float), w->stream));
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
  for (int b = 0; b < batch; ++b) ctx->probs_host.get()[b] = ctx->ws[b]->hp;
  CU(cudaMemcpyAsync(ctx->probs_dev.get(), ctx->probs_host.get(), sizeof(IcpProblem) * (size_t)batch, cudaMemcpyHostToDevice,
                     w0->stream));
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
  const IcpProblem* probs = ctx->probs_dev.get();
  int dynamic = batch > 1 ? 1 : 0;  // several problems: warps pull work from per-problem counters
  void* args[] = {(void*)&probs, (void*)&ctas, (void*)&dp, (void*)&dynamic};
  if (sharded) {  // narrow the staged problem to this shard's queries (cuts at cell starts, computed on the device)
    shard_slice_kernel<<<1, 32, 0, w0->stream>>>(ctx->probs_dev.get(), w0->job_dev, w0->hp.shard_rank, w0->hp.shard_count);
    LAUNCH_CHECK();
  }
  CU(cudaEventRecord(w0->ev_launch, w0->stream));
  CU(cudaLaunchCooperativeKernel((void*)icp_kernel, dim3(ctas * batch), dim3(kIcpThreads), args, kIcpPairBytes, w0->stream));
  ++ctx->launches;
  CU(cudaEventRecord(w0->ev2, w0->stream));
  // one gather and one copy for the whole batch (a pair of small copies per problem costs more than the kernel)
  collect_results_kernel<<<batch, 32, 0, w0->stream>>>(ctx->probs_dev.get(), ctx->results_dev.get());
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(ctx->results_host.get(), ctx->results_dev.get(), sizeof(IcpResult) * (size_t)batch, cudaMemcpyDeviceToHost,
                     w0->stream));
  return LS_OK;
}

// Device times of the last launch, recorded on workspace 0 (a batch is staged, built and launched as one, so its problems
// share them): staging .. end of the ICP launch, staging .. end of the build, the ICP launch.
void launch_times(ls_ctx* ctx, float t[3]) {
  const Workspace* w = ctx->ws[0];
  t[0] = t[1] = t[2] = 0.f;
  cudaEventElapsedTime(&t[0], w->ev0, w->ev2);
  cudaEventElapsedTime(&t[1], w->ev0, w->ev1);
  cudaEventElapsedTime(&t[2], w->ev_launch, w->ev2);
}

// After launch_icp + a synchronise of workspace 0's stream: unpack the results of problem k (workspace k).  `times`:
// launch_times of the launch, when the caller already has them.
int fetch_icp(ls_ctx* ctx, int k, int n, const float T0[16], float T_out[16], ls_icp_stats* stats,
              const float* times = nullptr) {
  const IcpResult& wk = ctx->results_host.get()[k];
  std::memcpy(T_out, wk.T_out, 16 * sizeof(float));
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->iterations = wk.iterations;
    stats->converged = wk.converged;
    stats->max_iter_reached = wk.max_iter_reached;
    stats->last_kept = wk.last_kept;
    stats->last_limit = wk.last_limit;
    stats->used_ratio = n > 0 ? (float)wk.last_kept / (float)n : 0.f;
    float own[3];
    if (!times) {
      launch_times(ctx, own);
      times = own;
    }
    stats->device_ms = times[0];
    stats->build_ms = times[1];
    stats->icp_ms = times[2];
    stats->grid_cells = wk.n_cells0;
    stats->grid_tables = wk.n_tab1;
    stats->grid_overflow = wk.overflow;
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
  if (opt_ids) CU(cudaMemcpyAsync(opt_ids, w->ids.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, w->stream));
  if (opt_d2) CU(cudaMemcpyAsync(opt_d2, w->d2_out.get(), (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  if (opt_T_hist)
    CU(cudaMemcpyAsync(opt_T_hist, w->T_hist.get(), (size_t)prm->max_iterations * 16 * sizeof(float), cudaMemcpyDeviceToHost,
                       w->stream));
  CU(cudaStreamSynchronize(w->stream));
  return fetch_icp(ctx, 0, n, T0, T_out, stats);
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
    parts.pts[p] = s->pts.get();
    parts.nrm[p] = s->nrm.get();
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
  w->work = ctx->work_pool.get() + index;
  w->job_dev = ctx->jobs_dev.get() + index;
  w->job_host = ctx->jobs_host.get() + index;
  bool ok = cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreate(&w->ev0) == cudaSuccess && cudaEventCreate(&w->ev1) == cudaSuccess &&
            cudaEventCreate(&w->ev2) == cudaSuccess && cudaEventCreate(&w->ev_launch) == cudaSuccess &&
            w->bs.reserve(1, 1) == cudaSuccess;
  if (!ok) return nullptr;  // partially built workspace is leaked only on an out-of-memory init failure
  return w;
}
void free_workspace(Workspace* w) {
  if (!w) return;
  if (w->stream) cudaStreamSynchronize(w->stream);
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
  if (ctx->probs_dev.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->probs_host.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->jobs_dev.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->jobs_host.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->work_pool.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->results_dev.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->results_host.reserve(kMaxBatch, kMaxBatch) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ctx->T0_dev.reserve(16, 16) != cudaSuccess) return bail(LS_ERR_NOMEM);
  if (ensure_workspaces(ctx, 1) != LS_OK) return bail(LS_ERR_NOMEM);
  *out = ctx;
  return LS_OK;
}

void ls_b200_destroy(ls_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (Workspace* w : ctx->ws) free_workspace(w);
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
  CU(cudaMemcpyAsync(ctx->reading.get(), reading4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->ref_stage.get(), ref4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if ((rc = upload_normals(ctx, w, ref_normals, normals_stride, m, ctx->ref_nrm_stage.get()))) return rc;
  Parts parts;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = 1;
  parts.offset[0] = 0;
  parts.offset[1] = m;
  parts.pts[0] = ctx->ref_stage.get();
  parts.nrm[0] = ctx->ref_nrm_stage.get();
  parts.identity[0] = 1;
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  return run_icp(ctx, prm, ctx->reading.get(), n, T0, T_out, stats, opt_ids, opt_d2, opt_T_iter_hist);
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
  CU(cudaMemcpyAsync(ctx->reading.get(), reading4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->ref_stage.get(), ref4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemsetAsync(ctx->ref_nrm_stage.get(), 0, (size_t)m * sizeof(float4), w->stream));
  Parts parts;
  std::memset(&parts, 0, sizeof(parts));
  parts.n_parts = 1;
  parts.offset[1] = m;
  parts.pts[0] = ctx->ref_stage.get();
  parts.nrm[0] = ctx->ref_nrm_stage.get();
  parts.identity[0] = 1;
  if ((rc = enqueue_build(ctx, w, parts, r, T0))) return rc;
  w->job_host->reading = ctx->reading.get();
  w->job_host->n = n;
  CU(cudaMemcpyAsync(w->job_dev, w->job_host, sizeof(BuildJob), cudaMemcpyHostToDevice, w->stream));
  reading_kernel<<<dim3(blocks_for(n, 256, ctx->sm_count * 8), 1), 256, 0, w->stream>>>(w->job_dev);
  LAUNCH_CHECK();
  GridView v{w->top.get(), w->tab1.get(), w->srt_pts.get(), w->pyr.get(), w->topmask.get()};
  nn_query_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->bs.get(), v, w->rd.get(), n, w->ids.get(),
                                                                                w->d2.get());
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(ids, w->ids.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, w->stream));
  CU(cudaMemcpyAsync(d2, w->d2.get(), (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
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
  CU(cudaMemcpyAsync(ctx->T0_dev.get(), T, 16 * sizeof(float), cudaMemcpyHostToDevice, w->stream));
  CU(cudaMemcpyAsync(ctx->reading.get(), in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if (normals && (rc = upload_normals(ctx, w, normals, normals_stride, n, ctx->ref_nrm_stage.get()))) return rc;
  transform_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(
      ctx->T0_dev.get(), ctx->reading.get(), normals ? ctx->ref_nrm_stage.get() : nullptr, n, w->rd.get(), w->sub_nrm.get());
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(out4, w->rd.get(), (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
  if (normals) {
    pack_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->sub_nrm.get(), n,
                                                                                         (float*)w->srt_nrm.get());
    LAUNCH_CHECK();
    CU(cudaMemcpyAsync(out_normals3, w->srt_nrm.get(), (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
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
    const size_t c = (size_t)max_pts_per_scan;
    if (s.pts.reserve(c, c) != cudaSuccess || s.nrm.reserve(c, c) != cudaSuccess ||
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
  for (auto& s : map->slots)
    if (s.ready) cudaEventDestroy(s.ready);
  for (int k = 0; k < kStageRing; ++k)
    if (map->stage_free[k]) cudaEventDestroy(map->stage_free[k]);
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
  if (map->host_stage[k].reserve(nf + nn, nf + nn + 1024) != cudaSuccess)
    return fail(ctx, LS_ERR_NOMEM, "pinned staging allocation failed");
  float* hf = map->host_stage[k].get();
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
    if (map->stage[k].reserve(need, need + 1024) != cudaSuccess) return fail(ctx, LS_ERR_NOMEM, "staging allocation failed");
    CU(cudaMemcpyAsync(s.pts.get(), features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, map->up_stream));
    CU(cudaMemcpyAsync(map->stage[k].get(), normals, need * sizeof(float), cudaMemcpyHostToDevice, map->up_stream));
    expand_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, map->up_stream>>>(map->stage[k].get(), normals_stride,
        n, s.nrm.get());
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
  GridView v{w->top.get(), w->tab1.get(), w->srt_pts.get(), w->pyr.get(), w->topmask.get()};
  knn_normals_kernel<<<blocks_for(n, 128, ctx->sm_count * 16), 128, 0, w->stream>>>(w->bs.get(), v, w->sub_pts.get(), n, knn,
                                                                                    nrm_out);
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
  CU(cudaMemcpyAsync(ctx->reading.get(), features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if ((rc = enqueue_normals(ctx, w, ctx->reading.get(), n, knn, ctx->ref_nrm_stage.get()))) return rc;
  pack_normals_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(ctx->ref_nrm_stage.get(), n,
                                                                                    (float*)w->srt_nrm.get());
  LAUNCH_CHECK();
  CU(cudaMemcpyAsync(out_normals3, w->srt_nrm.get(), (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
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
    CU(cudaMemcpyAsync(s.pts.get(), features4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
    int rc = enqueue_normals(ctx, w, s.pts.get(), n, knn, s.nrm.get());
    if (rc) return rc;
    CU(cudaStreamSynchronize(w->stream));
  }
  s.n = n;
  s.id = id;
  s.used = true;
  *scan_id = id;
  return LS_OK;
}

// ---- per-scan input filters -----------------------------------------------------------------------------------------
namespace {
bool chain_valid(const ls_point_filter* f, int n_filters) {
  if (n_filters < 0 || (n_filters > 0 && !f)) return false;
  for (int k = 0; k < n_filters; ++k)
    if (f[k].type < LS_PF_REMOVE_NAN || f[k].type > LS_PF_SAMPLING_SURFACE_NORMAL) return false;
  return true;
}
bool chain_makes_normals(const ls_point_filter* f, int n_filters) {
  for (int k = 0; k < n_filters; ++k)
    if (f[k].type == LS_PF_SURFACE_NORMAL || f[k].type == LS_PF_SAMPLING_SURFACE_NORMAL) return true;
  return false;
}

// Upload a host cloud (and its normals) into the chain buffers and run the chain on workspace 0's stream.  On return the
// result is in ctx->chain.pts[*cur].get() / nrm[*cur] (normals valid iff *has_nrm), *n_out points; nothing has been copied back
// but counts.  Runs of mask filters are one flag launch per point-wise run / sampler plus one compaction; the voxel grid
// and the normals work on the device buffers in place of ls_voxel_grid / ls_estimate_normals' host round trips.
int run_chain(ls_ctx* ctx, const ls_point_filter* f, int n_filters, const float* in4, const float* normals, int normals_stride,
              int n, int* cur, bool* has_nrm, int* n_out) {
  Workspace* w = ctx->ws[0];
  lsf::ChainBuffers& b = ctx->chain;
  CU(lsf::reserve(b, n));
  *cur = 0;
  *has_nrm = normals != nullptr;
  *n_out = n;
  if (n == 0) return LS_OK;
  int rc;
  CU(cudaMemcpyAsync(b.pts[0].get(), in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, w->stream));
  if (normals && (rc = upload_normals(ctx, w, normals, normals_stride, n, b.nrm[0].get()))) return rc;
  int k = 0, m = n, c = 0;
  while (k < n_filters && m > 0) {
    const ls_point_filter& fk = f[k];
    if (lsf::is_mask_filter(fk.type)) {
      int used = 0;
      CU(lsf::enqueue_mask_run(f + k, n_filters - k, b.pts[c].get(), *has_nrm ? b.nrm[c].get() : nullptr, m, b.pts[1 - c].get(),
                               b.nrm[1 - c].get(), b,
                               w->stream, &used, &ctx->launches));
      CU(cudaMemcpyAsync(&m, b.small.get() + 6, sizeof(int), cudaMemcpyDeviceToHost, w->stream));
      CU(cudaStreamSynchronize(w->stream));
      c = 1 - c;
      k += used;
    } else if (fk.type == LS_PF_VOXEL_GRID) {
      int v = 0;
      rc = lsf::enqueue_voxel_grid(b.pts[c].get(), *has_nrm ? b.nrm[c].get() : nullptr, m, fk.leaf, b.pts[1 - c].get(),
                                   b.nrm[1 - c].get(), 0,
                                   lsf::voxel_buffers(b), w->stream, &v, &ctx->launches);
      if (rc == LS_ERR_ARG) return fail(ctx, rc, "filter %d: voxel leaf too small for the cloud's extent", k);
      if (rc) return fail(ctx, rc, "filter %d: voxel grid: %s", k, cudaGetErrorString(cudaGetLastError()));
      m = v;
      c = 1 - c;
      ++k;
    } else {  // (Sampling)SurfaceNormal: exact k-NN normals of the current cloud, then the sampling of the Sampling variant
      const int knn = fk.knn < 3 ? 3 : (fk.knn > LS_KNN_MAX ? LS_KNN_MAX : fk.knn);
      if ((rc = enqueue_normals(ctx, w, b.pts[c].get(), m, knn, b.nrm[c].get()))) return rc;
      *has_nrm = true;
      if (fk.type == LS_PF_SAMPLING_SURFACE_NORMAL && fk.prob < 1.0f) {
        int used = 0;
        CU(lsf::enqueue_mask_run(&fk, 1, b.pts[c].get(), b.nrm[c].get(), m, b.pts[1 - c].get(), b.nrm[1 - c].get(), b, w->stream,
                                 &used,
                                 &ctx->launches));
        CU(cudaMemcpyAsync(&m, b.small.get() + 6, sizeof(int), cudaMemcpyDeviceToHost, w->stream));
        CU(cudaStreamSynchronize(w->stream));
        c = 1 - c;
      }
      ++k;
    }
  }
  for (; k < n_filters; ++k)  // the cloud is empty: a normal filter further on still defines (zero) normals
    if (f[k].type == LS_PF_SURFACE_NORMAL || f[k].type == LS_PF_SAMPLING_SURFACE_NORMAL) *has_nrm = true;
  *cur = c;
  *n_out = m;
  return LS_OK;
}
}  // namespace

int ls_filter_cloud(ls_ctx* ctx, const ls_point_filter* filters, int n_filters, const float* in4, const float* normals,
                    int normals_stride, int n, float* out4, float* out_normals3, int* n_out) {
  if (!ctx) return LS_ERR_ARG;
  BUSY_CHECK(ctx);
  if (!chain_valid(filters, n_filters) || !in4 || !out4 || !n_out || n < 0 || (normals && normals_stride < 3))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (out_normals3 && !normals && !chain_makes_normals(filters, n_filters))
    return fail(ctx, LS_ERR_ARG, "normals requested from a cloud without normals and a chain without a normal filter");
  *n_out = 0;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  int cur = 0, m = 0, rc;
  bool has_nrm = false;
  if ((rc = run_chain(ctx, filters, n_filters, in4, normals, normals_stride, n, &cur, &has_nrm, &m))) return rc;
  if (m > 0) {
    CU(cudaMemcpyAsync(out4, ctx->chain.pts[cur].get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
    if (out_normals3) {
      pack_normals_kernel<<<blocks_for(m, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(ctx->chain.nrm[cur].get(), m,
                                                                                           (float*)ctx->chain.nrm[1 - cur].get());
      LAUNCH_CHECK();
      CU(cudaMemcpyAsync(out_normals3, ctx->chain.nrm[1 - cur].get(), (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost,
                         w->stream));
    }
    CU(cudaStreamSynchronize(w->stream));
  }
  *n_out = m;
  return LS_OK;
}

int ls_map_push_scan_filtered(ls_map* map, const ls_point_filter* filters, int n_filters, const float* in4, const float* normals,
                              int normals_stride, int n, uint64_t* scan_id, int* n_kept) {
  if (!map) return LS_ERR_ARG;
  ls_ctx* ctx = map->ctx;
  BUSY_CHECK(ctx);
  if (!chain_valid(filters, n_filters) || !in4 || !scan_id || !n_kept || n < 0 || (normals && normals_stride < 3))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!normals && !chain_makes_normals(filters, n_filters))
    return fail(ctx, LS_ERR_ARG, "a scan without normals needs a normal filter in its chain (a slot must serve as a reference)");
  *n_kept = 0;
  CU(cudaSetDevice(ctx->device));
  Workspace* w = ctx->ws[0];
  int cur = 0, m = 0, rc;
  bool has_nrm = false;
  if ((rc = run_chain(ctx, filters, n_filters, in4, normals, normals_stride, n, &cur, &has_nrm, &m))) return rc;
  if (m > map->max_pts) return fail(ctx, LS_ERR_ARG, "the chain kept %d points, more than a slot holds (%d)", m, map->max_pts);
  // the batch in flight cannot read the slot this evicts: BUSY_CHECK above; an asynchronous upload into it may still run
  const uint64_t id = map->next_id++;
  ls_scan_slot& s = map->slots[id % (uint64_t)map->capacity];
  s.used = false;
  if (s.async) {
    CU(cudaEventSynchronize(s.ready));
    s.async = false;
  }
  if (m > 0) {
    CU(cudaMemcpyAsync(s.pts.get(), ctx->chain.pts[cur].get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToDevice, w->stream));
    CU(cudaMemcpyAsync(s.nrm.get(), ctx->chain.nrm[cur].get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToDevice, w->stream));
    CU(cudaStreamSynchronize(w->stream));
  }
  s.n = m;
  s.id = id;
  s.used = true;
  *scan_id = id;
  *n_kept = m;
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
  return run_icp(ctx, prm, rs->pts.get(), n, T0, T_out, stats, opt_ids, opt_d2, opt_T_iter_hist);
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
  if ((rc = prep_icp(ctx, w, prm, rs->pts.get(), n, T0, false, false))) return rc;
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
  ctx->xflag_base += ctx->results_host.get()[0].xsignals;
  return fetch_icp(ctx, 0, n, T0, T_out, stats);
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
  assemble_points_kernel<<<blocks_for(n, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(rd, ctx->reading.get());
  LAUNCH_CHECK();
  if ((rc = enqueue_build(ctx, w, ref, r, T0))) return rc;
  return run_icp(ctx, prm, ctx->reading.get(), n, T0, T_out, stats, nullptr, nullptr, nullptr);
}

// Several independent scan -> sub-map registrations in ONE cooperative launch (the multi-robot case: the
// reference's n_laser_slam_workers tracks, reference incremental_estimator.cpp:22-26, hosted on one GPU).
// Problem b stages on its own stream (assembly + hash build overlap across problems); the persistent kernel's
// grid is split into `batch` CTA groups, each with its own barrier, so one problem's barrier / solve latency is
// filled by the others' search.  Results are bit-identical to `batch` separate ls_icp_register_submap calls.
// A problem with an empty reading or an empty sub-map is not launched: like the single call it ends in
// LS_ERR_CONVERGENCE with T_out == T0, and the others run as if it were not there.
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
  const Resolved r = resolve(prm);
  ctx->pending_ws.assign(batch, -1);
  ctx->pending_T0.assign(T0s, T0s + 16 * (size_t)batch);
  ctx->pending_slots.clear();
  // validate every problem before anything is enqueued; the non-empty ones get workspaces 0.. in the caller's order
  int launched = 0;
  {
    int po = 0;
    for (int b = 0; b < batch; ++b) {
      if (n_parts[b] < 1 || n_parts[b] > kMaxParts) return fail(ctx, LS_ERR_ARG, "n_parts must be in [1,%d]", kMaxParts);
      const ls_scan_slot* rs = find_slot(map, reading_ids[b]);
      if (!rs) return fail(ctx, LS_ERR_STATE, "reading scan %llu is not resident", (unsigned long long)reading_ids[b]);
      ctx->pending_slots.emplace_back(map, (int)(rs - map->slots.data()));
      long long m = 0;
      for (int p = 0; p < n_parts[b]; ++p) {
        const ls_scan_slot* s = find_slot(map, part_ids[po + p]);
        if (!s) return fail(ctx, LS_ERR_STATE, "scan %llu is not resident (evicted or never pushed)", (unsigned long long)part_ids[po + p]);
        ctx->pending_slots.emplace_back(map, (int)(s - map->slots.data()));
        m += s->n;
      }
      if (rs->n > 0 && m > 0) ctx->pending_ws[b] = launched++;
      po += n_parts[b];
    }
  }
  ctx->pending_n.assign(launched, 0);
  ctx->pending_batch = batch;
  if (launched == 0) {  // every problem is empty: nothing to launch, _end reports LS_ERR_CONVERGENCE for each
    ctx->pending = true;
    return LS_OK;
  }
  if ((rc = ensure_workspaces(ctx, launched))) return rc;
  // stage every problem's job on the host, then ONE upload and ONE launch per build phase for the whole batch
  Workspace* w0 = ctx->ws[0];
  int n_max = 0, m_max = 0, part_off = 0;
  for (int b = 0; b < batch; ++b) {
    const int k = ctx->pending_ws[b];
    const int np = n_parts[b];
    part_off += np;
    if (k < 0) continue;
    Workspace* w = ctx->ws[k];
    const float* T0 = T0s + 16 * b;
    const ls_scan_slot* rs = find_slot(map, reading_ids[b]);
    Parts parts;
    if ((rc = make_parts(ctx, map, np, part_ids + (part_off - np), T_parts + 16 * (size_t)(part_off - np), &parts, w0->stream)))
      return rc;
    if (wait_slot(rs, w0->stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
    const int n = rs->n, m = parts.offset[np];
    ctx->pending_n[k] = n;
    n_max = n > n_max ? n : n_max;
    m_max = m > m_max ? m : m_max;
    if ((rc = ensure_capacity(ctx, w, n, m, r.max_cells, prm->max_iterations))) return rc;
    fill_job(w, parts, T0, rs->pts.get(), n);
    if ((rc = fill_problem(ctx, w, prm, n, T0, false, false))) return rc;
  }
  for (int k = 1; k < launched; ++k) {  // allocation-time clears a workspace enqueued on its own stream come first
    if (!ctx->ws[k]->stream_dirty) continue;
    CU(cudaEventRecord(ctx->ws[k]->ev2, ctx->ws[k]->stream));
    CU(cudaStreamWaitEvent(w0->stream, ctx->ws[k]->ev2, 0));
    ctx->ws[k]->stream_dirty = false;
  }
  CU(cudaEventRecord(w0->ev0, w0->stream));
  CU(cudaMemcpyAsync(ctx->jobs_dev.get(), ctx->jobs_host.get(), sizeof(BuildJob) * (size_t)launched, cudaMemcpyHostToDevice,
                     w0->stream));
  if ((rc = launch_build(ctx, ctx->jobs_dev.get(), launched, m_max, r, w0->stream))) return rc;
  if ((rc = launch_reading_sort(ctx, ctx->jobs_dev.get(), launched, n_max, r, w0->stream))) return rc;
  CU(cudaEventRecord(w0->ev1, w0->stream));
  CU(cudaMemsetAsync(ctx->work_pool.get(), 0, sizeof(IcpWork) * (size_t)launched, w0->stream));
  if ((rc = launch_icp(ctx, prm, launched, n_max))) return rc;
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
  float times[3] = {0.f, 0.f, 0.f};
  if (stats && !ctx->pending_n.empty()) launch_times(ctx, times);  // nothing was launched: no events to read
  for (int b = 0; b < batch; ++b) {
    const int k = ctx->pending_ws[b];
    if (k < 0) {  // not launched: T_out is already T0
      if (stats) std::memset(stats + b, 0, sizeof(*stats));
      statuses[b] = fail(ctx, LS_ERR_CONVERGENCE, "empty reading or reference");
      continue;
    }
    const int st = fetch_icp(ctx, k, ctx->pending_n[k], ctx->pending_T0.data() + 16 * b, T_outs + 16 * b,
                             stats ? stats + b : nullptr, times);
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
  CU(cudaMemcpyAsync(out4, w->sub_pts.get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
  if (out_normals3) {
    pack_normals_kernel<<<blocks_for(m, 256, ctx->sm_count * 8), 256, 0, w->stream>>>(w->sub_nrm.get(), m,
                                                                                         (float*)w->srt_nrm.get());
    LAUNCH_CHECK();
    CU(cudaMemcpyAsync(out_normals3, w->srt_nrm.get(), (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
  }
  CU(cudaStreamSynchronize(w->stream));
  return LS_OK;
}

}  // extern "C"

// ---- resident local map (LaserSlamWorker's map maintenance) -------------------------------------------------------------
// local[cur] is local_map_.  A filter crops it into local[1 - cur] and flips `cur`, so the old buffer is the snapshot
// without a copy; without a separate distant map that snapshot is also the filter's result and stays untouched until the
// next filter.  With one, the result is copied into `result` so later transforms and clears do not change it.
struct ls_local_map {
  ls_ctx* ctx = nullptr;
  ls_local_map_params prm{};
  int initial_cap = 0;
  cudaStream_t stream = nullptr;
  Buffer<float4> local[2];
  int cur = 0, n_local = 0;
  Buffer<float4> filt;  // local_map_filtered_
  int n_filt = 0;
  Buffer<float4> dist;  // distant_map_
  int n_dist = 0;
  Buffer<float4> queue;  // local_map_queue_, clouds back to back
  int n_queue = 0;
  std::vector<int> queue_sizes;
  Buffer<float4> result;  // the last filter's result (separate distant map only)
  int n_result = 0;
  lsf::ChainBuffers scratch;  // per-call flags, scans and voxel arrays, sized for the largest cloud seen
};

namespace {
// Grows a persistent cloud to hold `need` points (doubling), keeping its first `keep` points.  If the allocation fails the
// old buffer is left as it was.
int grow_cloud(ls_local_map* lm, Buffer<float4>& p, long long need, int keep) {
  ls_ctx* ctx = lm->ctx;
  const long long cap = (long long)p.capacity();
  if (need <= cap) return LS_OK;
  if (need > 0x7fffffffLL) return fail(ctx, LS_ERR_NOMEM, "local map cloud of %lld points", need);
  long long c = cap > lm->initial_cap ? cap : lm->initial_cap;
  while (c < need) c *= 2;
  if (c > 0x7fffffffLL) c = 0x7fffffffLL;
  Buffer<float4> q;
  if (q.reserve((size_t)c, (size_t)c) != cudaSuccess) return fail(ctx, LS_ERR_NOMEM, "local map growth to %lld points failed", c);
  if (keep > 0 &&
      cudaMemcpyAsync(q.get(), p.get(), (size_t)keep * sizeof(float4), cudaMemcpyDeviceToDevice, lm->stream) != cudaSuccess)
    return fail(ctx, LS_ERR_CUDA, "local map growth copy failed");
  CU(cudaStreamSynchronize(lm->stream));
  p = std::move(q);
  return LS_OK;
}

int reserve_scratch(ls_local_map* lm, int n) {
  ls_ctx* ctx = lm->ctx;
  const int want = n > lm->initial_cap ? n : lm->initial_cap;
  if (lm->scratch.pts[0].get() && (size_t)want <= lm->scratch.pts[0].capacity()) return LS_OK;
  CU(cudaStreamSynchronize(lm->stream));
  if (lsf::reserve(lm->scratch, want) != cudaSuccess)
    return fail(lm->ctx, LS_ERR_NOMEM, "local map scratch for %d points failed", want);
  return LS_OK;
}

// LS_LM_* -> (device pointer, points)
bool lm_cloud(const ls_local_map* lm, int which, const float4** p, int* n) {
  switch (which) {
    case LS_LM_LOCAL: *p = lm->local[lm->cur].get(); *n = lm->n_local; return true;
    case LS_LM_LOCAL_FILTERED: *p = lm->filt.get(); *n = lm->n_filt; return true;
    case LS_LM_DISTANT: *p = lm->dist.get(); *n = lm->n_dist; return true;
    case LS_LM_FILTERED_MAP:
      *p = lm->prm.separate_distant_map ? lm->result.get() : lm->local[1 - lm->cur].get();
      *n = lm->n_result;
      return true;
    case LS_LM_QUEUE: *p = lm->queue.get(); *n = lm->n_queue; return true;
    default: return false;
  }
}
}  // namespace

extern "C" {

int ls_local_map_create(ls_ctx* ctx, const ls_local_map_params* params, ls_local_map** out) {
  if (!ctx || !out) return LS_ERR_ARG;
  *out = nullptr;
  if (!params) return fail(ctx, LS_ERR_ARG, "bad argument");
  const ls_local_map_params& p = *params;
  if (!(p.distance_to_consider_fixed >= 0.0) || !((float)p.voxel_size_m > 0.0f) || !std::isfinite(p.voxel_size_m) ||
      p.minimum_point_number_per_voxel < 0 || !std::isfinite(p.ground_distance_to_robot_center_m))
    return fail(ctx, LS_ERR_ARG, "bad local map parameters (radius >= 0, leaf > 0, minimum >= 0)");
  CU(cudaSetDevice(ctx->device));
  ls_local_map* lm = new ls_local_map();
  lm->ctx = ctx;
  lm->prm = p;
  lm->initial_cap = p.initial_capacity_points > 0 ? p.initial_capacity_points : 262144;
  if (cudaStreamCreateWithFlags(&lm->stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    ls_local_map_destroy(lm);
    return fail(ctx, LS_ERR_NOMEM, "local map creation failed");
  }
  *out = lm;
  return LS_OK;
}

void ls_local_map_destroy(ls_local_map* lm) {
  if (!lm) return;
  cudaSetDevice(lm->ctx->device);
  if (lm->stream) cudaStreamSynchronize(lm->stream);
  if (lm->stream) cudaStreamDestroy(lm->stream);
  delete lm;
}

int ls_local_map_add_scan(ls_local_map* lm, const ls_map* ring, uint64_t scan_id, const float T_w_scan[16], double robot_z,
                          int* n_added) {
  if (!lm) return LS_ERR_ARG;
  ls_ctx* ctx = lm->ctx;
  if (!ring || !T_w_scan || !n_added) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (ring->ctx->device != ctx->device)
    return fail(ctx, LS_ERR_ARG, "the ring is on device %d, the local map on device %d", ring->ctx->device, ctx->device);
  CU(cudaSetDevice(ctx->device));
  const ls_scan_slot* s = find_slot(ring, scan_id);
  if (!s) return fail(ctx, LS_ERR_STATE, "scan %llu is not resident (evicted or never pushed)", (unsigned long long)scan_id);
  *n_added = 0;
  const int n = s->n;
  if (n == 0) return LS_OK;
  int rc;
  const int c = lm->cur;
  if ((rc = grow_cloud(lm, lm->local[c], (long long)lm->n_local + n, lm->n_local))) return rc;
  if ((rc = grow_cloud(lm, lm->queue, (long long)lm->n_queue + n, lm->n_queue))) return rc;
  if ((rc = reserve_scratch(lm, n))) return rc;
  if (wait_slot(s, lm->stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
  int kept = 0;
  const double z_min = robot_z - lm->prm.ground_distance_to_robot_center_m;
  rc = lsf::enqueue_local_map_append(s->pts.get(), n, T_w_scan, is_identity16(T_w_scan),
                                     lm->prm.remove_ground_from_local_map != 0, z_min, lm->local[c].get() + lm->n_local,
                                     lm->queue.get() + lm->n_queue, lm->scratch, lm->stream, &kept, &ctx->launches);
  if (rc) return fail(ctx, rc, "local map append failed");
  if (kept > 0) {
    lm->n_local += kept;
    lm->n_queue += kept;
    lm->queue_sizes.push_back(kept);
  }
  *n_added = kept;
  return LS_OK;
}

int ls_local_map_filter(ls_local_map* lm, const double center[3], int* n_filtered_map) {
  if (!lm) return LS_ERR_ARG;
  ls_ctx* ctx = lm->ctx;
  if (!center || !n_filtered_map) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  const bool separate = lm->prm.separate_distant_map != 0;
  const double radius = lm->prm.distance_to_consider_fixed, height = 40.0;  // the reference hard-codes the height
  const int c = lm->cur, n = lm->n_local;
  const float4* snap = lm->local[c].get();
  int rc;
  // every buffer this call can write, before anything changes (the previous result is kept until the new one exists)
  if ((rc = grow_cloud(lm, lm->local[1 - c], n, separate ? 0 : lm->n_result))) return rc;
  if ((rc = reserve_scratch(lm, n))) return rc;
  if (separate) {
    if ((rc = grow_cloud(lm, lm->filt, n, lm->n_filt))) return rc;
    if ((rc = grow_cloud(lm, lm->dist, (long long)lm->n_dist + n, lm->n_dist))) return rc;
    if ((rc = grow_cloud(lm, lm->result, (long long)lm->n_dist + 2LL * n, lm->n_result))) return rc;
  }
  int n_cropped = 0;
  if ((rc = lsf::enqueue_cylinder_crop(snap, n, center, radius, height, lm->local[1 - c].get(), lm->scratch, lm->stream,
                                       &n_cropped,
                                       &ctx->launches)))
    return fail(ctx, rc, "local map crop failed");
  if (!separate) {  // the result is the snapshot itself, uncropped and not voxelised
    lm->cur = 1 - c;
    lm->n_local = n_cropped;
    lm->n_result = n;
    *n_filtered_map = n;
    return LS_OK;
  }
  const float leaf[3] = {(float)lm->prm.voxel_size_m, (float)lm->prm.voxel_size_m, (float)lm->prm.voxel_size_m};
  lsf::VoxelBuffers vb = lsf::voxel_buffers(lm->scratch);
  vb.cent = lm->scratch.nrm[0].get();
  float4* vox = lm->scratch.pts[1].get();
  int m = 0;
  if ((rc = lsf::enqueue_voxel_grid(snap, nullptr, n, leaf, vox, nullptr, lm->prm.minimum_point_number_per_voxel, vb, lm->stream,
                                    &m, &ctx->launches)))
    return fail(ctx, rc, rc == LS_ERR_ARG ? "leaf too small for the local map's extent" : "local map voxel grid failed");
  int n_in = 0, n_out = 0;
  if ((rc = lsf::enqueue_cylinder_split(vox, m, center, radius, height, lm->filt.get(), lm->dist.get() + lm->n_dist, lm->scratch,
                                        lm->stream,
                                        &n_in, &n_out, &ctx->launches)))
    return fail(ctx, rc, "local map split failed");
  lm->cur = 1 - c;
  lm->n_local = n_cropped;
  lm->n_filt = n_in;
  lm->n_dist += n_out;
  if (n_in > 0) CU(cudaMemcpyAsync(lm->result.get(), lm->filt.get(), (size_t)n_in * sizeof(float4), cudaMemcpyDeviceToDevice,
                                   lm->stream));
  if (lm->n_dist > 0)
    CU(cudaMemcpyAsync(lm->result.get() + n_in, lm->dist.get(), (size_t)lm->n_dist * sizeof(float4), cudaMemcpyDeviceToDevice,
                       lm->stream));
  CU(cudaStreamSynchronize(lm->stream));
  lm->n_result = n_in + lm->n_dist;
  *n_filtered_map = lm->n_result;
  return LS_OK;
}

int ls_local_map_size(const ls_local_map* lm, int which) {
  if (!lm) return LS_ERR_ARG;
  const float4* p;
  int n;
  return lm_cloud(lm, which, &p, &n) ? n : LS_ERR_ARG;
}

int ls_local_map_download(const ls_local_map* lm, int which, float* out4, int cap, int* n_out) {
  if (!lm) return LS_ERR_ARG;
  ls_ctx* ctx = lm->ctx;
  const float4* p;
  int n;
  if (!n_out || !lm_cloud(lm, which, &p, &n)) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n > cap || (n > 0 && !out4)) return fail(ctx, LS_ERR_ARG, "buffer of %d points for a cloud of %d", cap, n);
  CU(cudaSetDevice(ctx->device));
  if (n > 0) CU(cudaMemcpyAsync(out4, p, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, lm->stream));
  CU(cudaStreamSynchronize(lm->stream));
  *n_out = n;
  return LS_OK;
}

int ls_local_map_take_queue(ls_local_map* lm, float* out4, int cap_points, int* cloud_offsets, int cap_clouds, int* n_clouds) {
  if (!lm) return LS_ERR_ARG;
  ls_ctx* ctx = lm->ctx;
  if (!cloud_offsets || !n_clouds) return fail(ctx, LS_ERR_ARG, "bad argument");
  const int k = (int)lm->queue_sizes.size();
  if (lm->n_queue > cap_points || k > cap_clouds || (lm->n_queue > 0 && !out4))
    return fail(ctx, LS_ERR_ARG, "buffers of %d points / %d clouds for a queue of %d / %d", cap_points, cap_clouds, lm->n_queue, k);
  CU(cudaSetDevice(ctx->device));
  if (lm->n_queue > 0)
    CU(cudaMemcpyAsync(out4, lm->queue.get(), (size_t)lm->n_queue * sizeof(float4), cudaMemcpyDeviceToHost, lm->stream));
  CU(cudaStreamSynchronize(lm->stream));
  cloud_offsets[0] = 0;
  for (int j = 0; j < k; ++j) cloud_offsets[j + 1] = cloud_offsets[j] + lm->queue_sizes[j];
  *n_clouds = k;
  lm->queue_sizes.clear();
  lm->n_queue = 0;
  return LS_OK;
}

int ls_local_map_transform(ls_local_map* lm, const float T[16]) {
  if (!lm) return LS_ERR_ARG;
  ls_ctx* ctx = lm->ctx;
  if (!T) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  float4* clouds[2] = {lm->local[lm->cur].get(), lm->filt.get()};
  const int counts[2] = {lm->n_local, lm->n_filt};
  for (int k = 0; k < 2; ++k) {
    const int rc = lsf::enqueue_transform_in_place(clouds[k], counts[k], T, lm->stream, &ctx->launches);
    if (rc) return fail(ctx, rc, "local map transform failed");
  }
  CU(cudaStreamSynchronize(lm->stream));
  return LS_OK;
}

int ls_local_map_clear(ls_local_map* lm) {
  if (!lm) return LS_ERR_ARG;
  lm->n_local = 0;
  lm->n_filt = 0;
  return LS_OK;
}

}  // extern "C"

// ---- resident occupancy map (laser_to_octomap's insertion loop; kernels in ls_occupancy.cu) ------------------------------
namespace {
// A stream and the two events that time work on it: start() .. stop(&ms).  The calls return the CUDA status for CU.
struct DeviceClock {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // All three or none: false, with whatever was created destroyed again, when one cannot be created.
  bool create() {
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) == cudaSuccess && cudaEventCreate(&ev0) == cudaSuccess &&
        cudaEventCreate(&ev1) == cudaSuccess)
      return true;
    cudaGetLastError();
    destroy();
    return false;
  }
  // The stream's work finishes first.
  void destroy() {
    if (stream) cudaStreamSynchronize(stream);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
    stream = nullptr, ev0 = ev1 = nullptr;
  }
  cudaError_t start() { return cudaEventRecord(ev0, stream); }
  // Waits for the work since start(); *ms: its device time.
  cudaError_t stop(float* ms) {
    cudaError_t e = cudaEventRecord(ev1, stream);
    if (e == cudaSuccess) e = cudaEventSynchronize(ev1);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, ev0, ev1);
    return e;
  }
};

constexpr uint64_t kNoVersion = ~0ull;
}  // namespace

struct ls_occupancy {
  ls_ctx* ctx = nullptr;
  lso::Params prm{};
  DeviceClock clock;
  lso::Map map;
  // Every change to the map increments `version`.  Each cached product below records the version it reflects (kNoVersion:
  // none) and is current while that equals `version`.
  uint64_t version = 0;
  // The last build of each tree format (indexed by lso::TreeFormat), cached apart.
  struct Tree {
    lso::Octree tree;
    uint64_t version = kNoVersion;
    float ms = 0.f;
  } trees[2];
  lso::Changes changes;  // change detection's baseline and scratch (ls_changes.cu)
  bool tracking = false;
  lso::Leaves leaves;  // the last leaf list (ls_occupancy_build_leaves)
  uint64_t leaves_version = kNoVersion;
  lso::Projection projection;  // the last 2D projection (ls_occupancy_build_projection)
  uint64_t projection_version = kNoVersion;
};

namespace {
using lso::TreeFormat;

ls_occupancy::Tree& tree_of(ls_occupancy* om, TreeFormat f) { return om->trees[(int)f]; }

// The error texts' name of a format: "octree" or "full octree".
const char* tree_name(TreeFormat f) { return f == TreeFormat::Full ? "full octree" : "octree"; }

int build_tree(ls_occupancy* om, TreeFormat f) {
  ls_ctx* ctx = om->ctx;
  ls_occupancy::Tree& t = tree_of(om, f);
  t.version = kNoVersion;
  CU(om->clock.start());
  const int rc = lso::build_tree(om->map, om->prm, f, t.tree, om->clock.stream, &ctx->launches);
  if (rc) return fail_lso(ctx, rc, f == TreeFormat::Full ? "full octree export" : "octree export");
  CU(om->clock.stop(&t.ms));
  t.version = om->version;
  return LS_OK;
}

// Makes the build of format f current, building it now unless it already is; *built: whether it was built now.
int current_tree(ls_occupancy* om, TreeFormat f, bool* built) {
  *built = tree_of(om, f).version != om->version;
  return *built ? build_tree(om, f) : LS_OK;
}

void full_stats(const ls_occupancy* om, ls_full_octree_stats* stats) {
  if (!stats) return;
  const ls_occupancy::Tree& t = om->trees[(int)TreeFormat::Full];
  stats->nodes = t.tree.nodes;
  stats->leaves = t.tree.leaves;
  stats->payload_bytes = t.tree.bytes;
  stats->device_ms = t.ms;
}

// The file at `path`, whole.  NULL on success, else why not.
const char* read_file(const char* path, std::vector<uint8_t>* data) {
  FILE* f = std::fopen(path, "rb");
  if (!f) return "cannot open the file";
  uint8_t buf[1 << 16];
  size_t got;
  while ((got = std::fread(buf, 1, sizeof buf, f)) > 0) data->insert(data->end(), buf, buf + got);
  const bool err = std::ferror(f) != 0;
  std::fclose(f);
  return err ? "reading the file failed" : nullptr;
}

void octree_stats(const ls_occupancy* om, ls_octree_stats* stats) {
  if (!stats) return;
  const ls_occupancy::Tree& t = om->trees[(int)TreeFormat::Binary];
  stats->nodes = t.tree.nodes;
  stats->payload_bytes = t.tree.bytes;
  stats->occupied_leaves = t.tree.leaves;
  stats->device_ms = t.ms;
}

// A .bt header (with `full`, a .ot header) as laser_slam_b200.read_octomap (read_octomap_full) parses it: the first line
// exactly (a trailing \r dropped), then "#" and blank lines skipped, "key value" lines, up to "data"; id OcTree, an integer
// size >= 0 and a res.  *off: the payload's first byte.  NULL when it is valid, else why not.
const char* parse_bt_header(const std::vector<uint8_t>& d, size_t* off, long long* nodes, double* res, bool full = false) {
  size_t pos = 0;
  std::string line;
  auto next = [&]() {
    const uint8_t* nl = static_cast<const uint8_t*>(std::memchr(d.data() + pos, '\n', d.size() - pos));
    if (!nl) return false;
    const size_t end = (size_t)(nl - d.data());
    line.assign(reinterpret_cast<const char*>(d.data()) + pos, end - pos);
    pos = end + 1;
    while (!line.empty() && line.back() == '\r') line.pop_back();
    return true;
  };
  auto strip = [](const std::string& s) {
    const char* ws = " \t\n\r\v\f";
    const size_t a = s.find_first_not_of(ws);
    return a == std::string::npos ? std::string() : s.substr(a, s.find_last_not_of(ws) + 1 - a);
  };
  if (d.empty() || !next()) return "header ends early";
  if (line != (full ? "# Octomap OcTree file" : "# Octomap OcTree binary file"))
    return full ? "not an octomap full tree file (first line)" : "not an octomap binary file (first line)";
  std::string id, size, resolution;
  bool have_id = false, have_size = false, have_res = false;
  for (;;) {
    if (!next()) return "header ends early";
    if ((!line.empty() && line[0] == '#') || strip(line).empty()) continue;
    if (line == "data") break;
    const size_t sp = line.find(' ');
    const std::string key = line.substr(0, sp), value = sp == std::string::npos ? std::string() : strip(line.substr(sp + 1));
    if (key == "id") id = value, have_id = true;
    if (key == "size") size = value, have_size = true;
    if (key == "res") resolution = value, have_res = true;
  }
  if (!have_id || id != "OcTree") return "tree type is not OcTree";
  if (!have_size || !have_res || size.empty() || resolution.empty()) return "bad or missing size / res line";
  char* e = nullptr;
  errno = 0;
  const long long n = std::strtoll(size.c_str(), &e, 10);
  if (*e != '\0' || errno == ERANGE) return "bad or missing size / res line";
  const double r = std::strtod(resolution.c_str(), &e);
  if (*e != '\0') return "bad or missing size / res line";
  if (n < 0) return "negative size";
  *off = pos, *nodes = n, *res = r;
  return nullptr;
}
int download_tree(ls_occupancy* om, TreeFormat f, uint8_t* payload, int64_t payload_cap, float* centres4, uint8_t* depths,
                  int64_t leaf_cap) {
  ls_ctx* ctx = om->ctx;
  if (tree_of(om, f).version != om->version)
    return fail(ctx, LS_ERR_STATE, f == TreeFormat::Full ? "no current full octree: build it after the last insert or read"
                                                         : "no current octree: build it after the last insert");
  const lso::Octree& t = tree_of(om, f).tree;
  if ((t.bytes > 0 && !payload) || payload_cap < t.bytes)
    return fail(ctx, LS_ERR_ARG, "a payload buffer of %lld bytes for %lld", (long long)payload_cap, t.bytes);
  if ((centres4 || depths) && leaf_cap < t.leaves)
    return fail(ctx, LS_ERR_ARG, "leaf buffers of %lld for %lld occupied leaves", (long long)leaf_cap, t.leaves);
  CU(cudaSetDevice(ctx->device));
  const int rc = lso::download_octree(t, payload, centres4, depths, om->clock.stream);
  if (rc) return fail(ctx, rc, "%s download failed", tree_name(f));
  return LS_OK;
}

// octomap's writeBinaryConst (.bt) or AbstractOcTree::write (.ot): the header, then the payload of the current build
int write_tree(ls_occupancy* om, TreeFormat f, const char* path) {
  ls_ctx* ctx = om->ctx;
  if (!path) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  bool built;
  int rc = current_tree(om, f, &built);
  if (rc) return rc;
  const ls_occupancy::Tree& t = tree_of(om, f);
  std::vector<uint8_t> payload((size_t)t.tree.bytes);
  if ((rc = lso::download_octree(t.tree, payload.data(), nullptr, nullptr, om->clock.stream)))
    return fail(ctx, rc, "%s download failed", tree_name(f));
  // the resolution as a default std::ostream prints a double (%g)
  char head[256];
  const int n = std::snprintf(head, sizeof head,
                              "%s\n# (feel free to add / change comments, but leave the first line as it is!)\n#\nid OcTree\n"
                              "size %lld\nres %g\ndata\n",
                              f == TreeFormat::Full ? "# Octomap OcTree file" : "# Octomap OcTree binary file", t.tree.nodes,
                              om->prm.res);
  FILE* file = std::fopen(path, "wb");
  if (!file) return fail(ctx, LS_ERR_ARG, "cannot open %s for writing", path);
  bool ok = std::fwrite(head, 1, (size_t)n, file) == (size_t)n;
  if (ok && !payload.empty()) ok = std::fwrite(payload.data(), 1, payload.size(), file) == payload.size();
  ok = std::fclose(file) == 0 && ok;
  if (!ok) return fail(ctx, LS_ERR_ARG, "writing %s failed", path);
  return LS_OK;
}

int read_tree(ls_occupancy* om, TreeFormat f, const uint8_t* payload, int64_t payload_bytes, int64_t nodes, double resolution,
              ls_octomap_read_stats* stats) {
  ls_ctx* ctx = om->ctx;
  if (nodes < 0 || payload_bytes < 0 || (payload_bytes > 0 && !payload)) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!(resolution > 0.0) || !std::isfinite(resolution))
    return fail(ctx, LS_ERR_ARG, "octomap resolution %g (finite and > 0)", resolution);
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  lso::Params P = om->prm;
  P.res = resolution;
  P.inv = 1.0 / resolution;
  lso::ReadCounters c;
  const char* why = "";
  const int rc = lso::read_tree(om->map, P, f, payload, payload_bytes, nodes, &c, &why, om->clock.stream, &ctx->launches);
  if (rc)
    return fail(ctx, rc, "octomap %sread refused, the map is unchanged: %s", f == TreeFormat::Full ? "full tree " : "", why);
  om->prm = P;
  ++om->version;
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  if (stats) {
    stats->nodes = (int64_t)c.nodes;
    stats->inner_nodes = (int64_t)c.inner;
    stats->free_leaves = (int64_t)c.free_leaves;
    stats->occupied_leaves = (int64_t)c.occ_leaves;
    stats->known_voxels = om->map.n_known;
    stats->bricks = om->map.pool_n;
    stats->resolution = P.res;
    stats->device_ms = ms;
  }
  return LS_OK;
}

int read_tree_file(ls_occupancy* om, TreeFormat f, const char* path, ls_octomap_read_stats* stats) {
  ls_ctx* ctx = om->ctx;
  if (!path) return fail(ctx, LS_ERR_ARG, "bad argument");
  std::vector<uint8_t> data;
  const char* why = read_file(path, &data);
  if (why) return fail(ctx, LS_ERR_ARG, "%s: %s", path, why);
  size_t off = 0;
  long long nodes = 0;
  double res = 0.0;
  why = parse_bt_header(data, &off, &nodes, &res, f == TreeFormat::Full);
  if (why) return fail(ctx, LS_ERR_ARG, "%s: %s", path, why);
  return read_tree(om, f, data.data() + off, (int64_t)(data.size() - off), nodes, res, stats);
}
}  // namespace

extern "C" {

void ls_occupancy_default_params(ls_occupancy_params* out) {
  if (!out) return;
  out->resolution = 0.075;  // laser_to_octomap.cpp:18-21
  out->prob_hit = 0.9;
  out->prob_miss = 0.4;
  out->max_range = 20.0;
  out->clamp_min = 0.12;  // volumetric_mapping's defaults
  out->clamp_max = 0.97;
  out->occupancy_threshold = 0.7;
  out->initial_capacity = 0;
}

int ls_occupancy_create(ls_ctx* ctx, const ls_occupancy_params* params, ls_occupancy** out) {
  if (!ctx || !out) return LS_ERR_ARG;
  *out = nullptr;
  if (!params) return fail(ctx, LS_ERR_ARG, "bad argument");
  const ls_occupancy_params& p = *params;
  auto prob = [](double x) { return x > 0.0 && x < 1.0; };
  if (!(p.resolution > 0.0) || !std::isfinite(p.resolution) || !prob(p.prob_hit) || !prob(p.prob_miss) || !prob(p.clamp_min) ||
      !prob(p.clamp_max) || !prob(p.occupancy_threshold) || !(p.clamp_min <= p.clamp_max) || std::isnan(p.max_range))
    return fail(ctx, LS_ERR_ARG, "bad occupancy map parameters (resolution > 0, probabilities in (0, 1), clamp_min <= clamp_max)");
  CU(cudaSetDevice(ctx->device));
  auto logodds = [](double x) { return (float)std::log(x / (1.0 - x)); };
  ls_occupancy* om = new ls_occupancy();
  om->ctx = ctx;
  om->prm = lso::Params{p.resolution, 1.0 / p.resolution, p.max_range, logodds(p.prob_hit), logodds(p.prob_miss),
                        logodds(p.clamp_min), logodds(p.clamp_max), logodds(p.occupancy_threshold)};
  int bricks = 32768;
  if (p.initial_capacity > 0) bricks = p.initial_capacity < (1 << 24) ? p.initial_capacity : (1 << 24);
  const int rc = om->clock.create() ? lso::init(om->map, bricks, om->clock.stream) : LS_ERR_NOMEM;
  if (rc) {
    ls_occupancy_destroy(om);
    return fail(ctx, rc, "occupancy map creation failed");
  }
  *out = om;
  return LS_OK;
}

void ls_occupancy_destroy(ls_occupancy* om) {
  if (!om) return;
  cudaSetDevice(om->ctx->device);
  om->clock.destroy();
  delete om;
}

int ls_occupancy_insert_scan(ls_occupancy* om, const ls_map* ring, uint64_t scan_id, const float T_w_scan[16],
                             ls_occupancy_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!ring || !T_w_scan) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (ring->ctx->device != ctx->device)
    return fail(ctx, LS_ERR_ARG, "the ring is on device %d, the occupancy map on device %d", ring->ctx->device, ctx->device);
  CU(cudaSetDevice(ctx->device));
  const ls_scan_slot* s = find_slot(ring, scan_id);
  if (!s) return fail(ctx, LS_ERR_STATE, "scan %llu is not resident (evicted or never pushed)", (unsigned long long)scan_id);
  if (wait_slot(s, om->clock.stream) != LS_OK) return fail(ctx, LS_ERR_CUDA, "cudaStreamWaitEvent failed");
  CU(om->clock.start());
  ++om->version;  // before the insert: a failed one may have changed voxels
  lso::Counters c;
  const int rc = lso::insert(om->map, om->prm, s->pts.get(), s->n, T_w_scan, is_identity16(T_w_scan), om->clock.stream,
                             &c, &ctx->launches);
  if (rc) return fail(ctx, rc, rc == LS_ERR_NOMEM ? "occupancy map growth failed" : "occupancy map insert failed");
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  if (stats) {
    stats->rays_cast = c.rays_cast;
    stats->rays_skipped = c.rays_skipped;
    stats->free_updates = (int64_t)c.free_upd;
    stats->occupied_updates = (int64_t)c.occ_upd;
    stats->known_voxels = om->map.n_known;
    stats->bricks = om->map.pool_n;
    stats->device_bytes = (int64_t)lso::device_bytes(om->map);
    stats->device_ms = ms;
  }
  return LS_OK;
}

int ls_occupancy_size(ls_occupancy* om, int which, int64_t* n) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n || (which != LS_OCC_KNOWN && which != LS_OCC_OCCUPIED)) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  long long m = 0;
  const int rc = lso::count(om->map, om->prm, which, &m, om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "occupancy map count failed");
  *n = m;
  return LS_OK;
}

int ls_occupancy_download(ls_occupancy* om, int which, uint64_t* keys, float* log_odds, float* centres4, int64_t cap,
                          int64_t* n) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n || (which != LS_OCC_KNOWN && which != LS_OCC_OCCUPIED)) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  long long m = 0;
  int rc = lso::count(om->map, om->prm, which, &m, om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "occupancy map count failed");
  if (m > cap) return fail(ctx, LS_ERR_ARG, "buffers of %lld voxels for %lld", (long long)cap, m);
  rc = lso::download(om->map, om->prm, which, m, keys, log_odds, centres4, om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "occupancy map download failed");
  *n = m;
  return LS_OK;
}

int ls_occupancy_build_octree(ls_occupancy* om, ls_octree_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  CU(cudaSetDevice(ctx->device));
  const int rc = build_tree(om, TreeFormat::Binary);
  if (!rc) octree_stats(om, stats);
  return rc;
}

int ls_occupancy_download_octree(ls_occupancy* om, uint8_t* payload, int64_t payload_cap, float* centres4, uint8_t* depths,
                                 int64_t leaf_cap) {
  if (!om) return LS_ERR_ARG;
  return download_tree(om, TreeFormat::Binary, payload, payload_cap, centres4, depths, leaf_cap);
}

int ls_occupancy_write_octomap(ls_occupancy* om, const char* path, ls_octree_stats* stats) {
  if (!om) return LS_ERR_ARG;
  const int rc = write_tree(om, TreeFormat::Binary, path);
  if (!rc) octree_stats(om, stats);
  return rc;
}

int ls_occupancy_read_octree(ls_occupancy* om, const uint8_t* payload, int64_t payload_bytes, int64_t nodes,
                             double resolution, ls_octomap_read_stats* stats) {
  if (!om) return LS_ERR_ARG;
  return read_tree(om, TreeFormat::Binary, payload, payload_bytes, nodes, resolution, stats);
}

int ls_occupancy_read_octomap(ls_occupancy* om, const char* path, ls_octomap_read_stats* stats) {
  if (!om) return LS_ERR_ARG;
  return read_tree_file(om, TreeFormat::Binary, path, stats);
}

int ls_occupancy_build_full_octree(ls_occupancy* om, ls_full_octree_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  CU(cudaSetDevice(ctx->device));
  const int rc = build_tree(om, TreeFormat::Full);
  if (!rc) full_stats(om, stats);
  return rc;
}

int ls_occupancy_download_full_octree(ls_occupancy* om, uint8_t* payload, int64_t payload_cap) {
  if (!om) return LS_ERR_ARG;
  return download_tree(om, TreeFormat::Full, payload, payload_cap, nullptr, nullptr, 0);
}

int ls_occupancy_write_octomap_full(ls_occupancy* om, const char* path, ls_full_octree_stats* stats) {
  if (!om) return LS_ERR_ARG;
  const int rc = write_tree(om, TreeFormat::Full, path);
  if (!rc) full_stats(om, stats);
  return rc;
}

int ls_occupancy_read_full_octree(ls_occupancy* om, const uint8_t* payload, int64_t payload_bytes, int64_t nodes,
                                  double resolution, ls_octomap_read_stats* stats) {
  if (!om) return LS_ERR_ARG;
  return read_tree(om, TreeFormat::Full, payload, payload_bytes, nodes, resolution, stats);
}

int ls_occupancy_read_octomap_full(ls_occupancy* om, const char* path, ls_octomap_read_stats* stats) {
  if (!om) return LS_ERR_ARG;
  return read_tree_file(om, TreeFormat::Full, path, stats);
}

}  // extern "C"

namespace {
// The query's device time (the map's clock, started before it) and its keys visited into *stats.
int query_done(ls_occupancy* om, long long visited, ls_occupancy_query_stats* stats) {
  ls_ctx* ctx = om->ctx;
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  if (stats) {
    stats->keys_visited = visited;
    stats->device_ms = ms;
  }
  return LS_OK;
}

void query_none(ls_occupancy_query_stats* stats) {
  if (stats) stats->keys_visited = 0, stats->device_ms = 0.f;
}
}  // namespace

extern "C" {

int ls_occupancy_cell_status(ls_occupancy* om, const double* points3, int n, int8_t* status, float* log_odds,
                             ls_occupancy_query_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n < 0 || (n > 0 && (!points3 || !status))) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n == 0) return query_none(stats), LS_OK;
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long visited = 0;
  const int rc = lso::query_cells(om->map, om->prm, points3, n, status, log_odds, &visited, om->clock.stream, &ctx->launches);
  if (rc) return fail_lso(ctx, rc, "cell query");
  return query_done(om, visited, stats);
}

int ls_occupancy_line_status(ls_occupancy* om, const double* starts3, const double* ends3, int n, const double* box3,
                             int stop_at_unknown, int8_t* status, uint64_t* first_keys, ls_occupancy_query_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n < 0 || (n > 0 && (!starts3 || !ends3 || !status))) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (box3)
    for (int a = 0; a < 3; ++a)
      if (!std::isfinite(box3[a]) || box3[a] < 0.0)
        return fail(ctx, LS_ERR_ARG, "bounding box size %g on axis %d (finite and >= 0)", box3[a], a);
  if (n == 0) return query_none(stats), LS_OK;
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long visited = 0;
  const int rc = lso::query_lines(om->map, om->prm, starts3, ends3, n, box3, stop_at_unknown, status, first_keys, &visited,
                                  om->clock.stream, &ctx->launches);
  if (rc == LS_ERR_ARG) return fail(ctx, rc, "%d segments with this bounding box make more than 2^31 - 1 lines", n);
  if (rc) return fail_lso(ctx, rc, "line query");
  return query_done(om, visited, stats);
}

int ls_occupancy_cast_rays(ls_occupancy* om, const float* origins3, const float* directions3, int n, int ignore_unknown,
                           double max_range, int8_t* result, float* ends3, ls_occupancy_query_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n < 0 || (n > 0 && (!origins3 || !directions3 || !result))) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n == 0) return query_none(stats), LS_OK;
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long visited = 0;
  const int rc = lso::query_rays(om->map, om->prm, origins3, directions3, n, ignore_unknown, max_range, result, ends3, &visited,
                                 om->clock.stream, &ctx->launches);
  if (rc) return fail_lso(ctx, rc, "ray query");
  return query_done(om, visited, stats);
}

int ls_occupancy_box_status(ls_occupancy* om, const double* centres3, const double* sizes3, int n, int8_t* status,
                            ls_occupancy_query_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n < 0 || (n > 0 && (!centres3 || !sizes3 || !status))) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n == 0) return query_none(stats), LS_OK;
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long visited = 0;
  const int rc = lso::box_status(om->map, om->prm, centres3, sizes3, n, status, &visited, om->clock.stream, &ctx->launches);
  if (rc == LS_ERR_ARG)
    return fail(ctx, rc, "box status refused: a size is negative or not finite, a box axis has more than 2^17 loop points, "
                         "or the boxes span more than 2^36 (box, brick) items");
  if (rc) return fail_lso(ctx, rc, "box status");
  return query_done(om, visited, stats);
}

int ls_occupancy_check_paths(ls_occupancy* om, const double* positions3, const int64_t* offsets, int n_paths,
                             const double robot_size3[3], int unknown_as_occupied, int64_t* first_collision,
                             ls_occupancy_query_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n_paths < 0 || (n_paths > 0 && (!offsets || !robot_size3 || !first_collision)))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (n_paths == 0) return query_none(stats), LS_OK;
  for (int a = 0; a < 3; ++a)  // checked here too, so a call whose paths are all empty refuses a bad size as well
    if (!std::isfinite(robot_size3[a]) || robot_size3[a] < 0.0)
      return fail(ctx, LS_ERR_ARG, "robot size %g on axis %d (finite and >= 0)", robot_size3[a], a);
  if (offsets[0] != 0) return fail(ctx, LS_ERR_ARG, "path offsets start at %lld, not 0", (long long)offsets[0]);
  for (int p = 0; p < n_paths; ++p)
    if (offsets[p + 1] < offsets[p]) return fail(ctx, LS_ERR_ARG, "path offsets decrease at path %d", p);
  if (offsets[n_paths] > 0x7fffffffLL) return fail(ctx, LS_ERR_ARG, "%lld poses (at most 2^31 - 1)", (long long)offsets[n_paths]);
  if (offsets[n_paths] > 0 && !positions3) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long visited = 0;
  const int rc = lso::check_paths(om->map, om->prm, positions3, offsets, n_paths, robot_size3, unknown_as_occupied,
                                  first_collision, &visited, om->clock.stream, &ctx->launches);
  if (rc == LS_ERR_ARG)
    return fail(ctx, rc, "path check refused: the robot box has more than 2^17 loop points on an axis, or the poses span "
                         "more than 2^36 (box, brick) items");
  if (rc) return fail_lso(ctx, rc, "path check");
  return query_done(om, visited, stats);
}

}  // extern "C"

namespace {
// A box centre and size: finite, the size >= 0.  NULL when valid, else why not.
const char* bad_box(const double* c3, const double* s3) {
  for (int a = 0; a < 3; ++a) {
    if (!std::isfinite(c3[a])) return "a box centre is not finite";
    if (!std::isfinite(s3[a]) || s3[a] < 0.0) return "a box size is not finite and >= 0";
  }
  return nullptr;
}
}  // namespace

extern "C" {

int ls_occupancy_set_boxes(ls_occupancy* om, const double* centres3, const double* sizes3, const int8_t* occupied, int n,
                           ls_occupancy_edit_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (n < 0 || (n > 0 && (!centres3 || !sizes3 || !occupied))) return fail(ctx, LS_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    const char* why = bad_box(centres3 + 3 * (size_t)i, sizes3 + 3 * (size_t)i);
    if (why) return fail(ctx, LS_ERR_ARG, "box %d: %s", i, why);
  }
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  long long set = 0, added = 0;
  const char* why = "";
  const int rc = lso::set_boxes(om->map, om->prm, centres3, sizes3, occupied, n, &set, &added, &why, om->clock.stream,
                                &ctx->launches);
  if (rc) return fail(ctx, rc, "set boxes refused, the map's voxels are unchanged: %s", why);
  if (set > 0) ++om->version;
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  if (stats) {
    stats->voxels_set = set;
    stats->new_known = added;
    stats->known_voxels = om->map.n_known;
    stats->bricks = om->map.pool_n;
    stats->device_bytes = (int64_t)lso::device_bytes(om->map);
    stats->device_ms = ms;
  }
  return LS_OK;
}

int ls_occupancy_clear(ls_occupancy* om) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  CU(cudaSetDevice(ctx->device));
  const int rc = lso::clear(om->map, om->clock.stream);
  ++om->version;
  if (rc) return fail(ctx, rc, "occupancy map reset failed");
  return LS_OK;
}

int ls_occupancy_box_voxels(ls_occupancy* om, const double center3[3], const double size3[3], int which, uint64_t* keys,
                            float* log_odds, float* centres4, int64_t cap, int64_t* n) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n) return fail(ctx, LS_ERR_ARG, "bad argument");
  *n = 0;
  if (!center3 || !size3 || cap < 0 || (which != LS_OCC_KNOWN && which != LS_OCC_OCCUPIED))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  const char* why = bad_box(center3, size3);
  if (why) return fail(ctx, LS_ERR_ARG, "%s", why);
  CU(cudaSetDevice(ctx->device));
  long long m = 0;
  const int rc = lso::box_voxels(om->map, om->prm, center3, size3, which, keys, log_odds, centres4, cap, &m, om->clock.stream,
                                 &ctx->launches);
  *n = m;
  if (rc == LS_ERR_ARG && m > cap) return fail(ctx, rc, "buffers of %lld voxels for %lld", (long long)cap, m);
  if (rc == LS_ERR_ARG) return fail(ctx, rc, "the box has more than 2^17 loop points on an axis or 2^31 - 1 in all");
  if (rc) return fail_lso(ctx, rc, "box voxels");
  return LS_OK;
}

int ls_occupancy_bounds(ls_occupancy* om, double min3[3], double max3[3]) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!min3 || !max3) return fail(ctx, LS_ERR_ARG, "bad argument");
  CU(cudaSetDevice(ctx->device));
  int kmin[3], kmax[3];
  bool empty = true;
  const int rc = lso::key_bounds(om->map, kmin, kmax, &empty, om->clock.stream, &ctx->launches);
  if (rc) return fail_lso(ctx, rc, "bounds");
  const double res = om->prm.res;
  for (int a = 0; a < 3; ++a) {
    // octomap's calcMinMax over depth-16 leaves: the lower corner, and the lower corner plus the voxel size
    min3[a] = empty ? 0.0 : (double)lso::centre_of(kmin[a], res) - res / 2.0;
    max3[a] = empty ? 0.0 : ((double)lso::centre_of(kmax[a], res) - res / 2.0) + res;
  }
  return LS_OK;
}

}  // extern "C"

namespace {
// The key of a region corner in double (lso::key_of's floor and offset), clamped to [0, 65535] instead of refused.
int clamped_key(double inv, double c) {
  const double s = std::floor(c * inv) + (double)lso::kKeyOffset;
  return s < 0.0 ? 0 : s > 65535.0 ? 65535 : (int)s;
}
}  // namespace

extern "C" {

int ls_occupancy_build_leaves(ls_occupancy* om, const double* region_min3, const double* region_max3, ls_leaf_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!region_min3 != !region_max3) return fail(ctx, LS_ERR_ARG, "a region needs both corners");
  int kmin[3] = {0, 0, 0}, kmax[3] = {65535, 65535, 65535};
  if (region_min3) {
    for (int a = 0; a < 3; ++a) {
      if (!std::isfinite(region_min3[a]) || !std::isfinite(region_max3[a]))
        return fail(ctx, LS_ERR_ARG, "region axis %d is not finite", a);
      if (region_min3[a] > region_max3[a]) return fail(ctx, LS_ERR_ARG, "region axis %d is inverted (min > max)", a);
      kmin[a] = clamped_key(om->prm.inv, region_min3[a]);
      kmax[a] = clamped_key(om->prm.inv, region_max3[a]);
    }
  }
  CU(cudaSetDevice(ctx->device));
  om->leaves_version = kNoVersion;
  bool built;
  int rc = current_tree(om, TreeFormat::Full, &built);
  if (rc) return rc;
  ls_occupancy::Tree& t = tree_of(om, TreeFormat::Full);
  CU(om->clock.start());
  rc = lso::build_leaves(om->map, om->prm, t.tree, kmin, kmax, om->leaves, om->clock.stream, &ctx->launches);
  if (rc) return fail_lso(ctx, rc, "leaf list");
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  om->leaves_version = om->version;
  if (stats) {
    const lso::Leaves& L = om->leaves;
    stats->free_leaves = L.n - L.n_occupied;
    stats->occupied_leaves = L.n_occupied;
    for (int d = 0; d < 17; ++d) stats->free_by_depth[d] = L.free[d], stats->occupied_by_depth[d] = L.occupied[d];
    stats->device_ms = ms + (built ? t.ms : 0.f);
  }
  return LS_OK;
}

int ls_occupancy_download_leaves(ls_occupancy* om, int which, float* centres4, uint8_t* depths, int8_t* states, int64_t cap,
                                 int64_t* n) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n) return fail(ctx, LS_ERR_ARG, "bad argument");
  *n = 0;
  if (cap < 0 || (which != LS_LEAVES_FREE && which != LS_LEAVES_OCCUPIED && which != LS_LEAVES_ALL) ||
      (cap > 0 && (!centres4 || !depths || !states)))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (om->leaves_version != om->version)
    return fail(ctx, LS_ERR_STATE, "no current leaf list: build it after the last change to the map");
  const lso::Leaves& L = om->leaves;
  const long long m = which == LS_LEAVES_ALL ? L.n : which == LS_LEAVES_OCCUPIED ? L.n_occupied : L.n - L.n_occupied;
  *n = m;
  if (m > cap) return fail(ctx, LS_ERR_ARG, "buffers of %lld leaves for %lld", (long long)cap, m);
  if (m == 0) return LS_OK;
  CU(cudaSetDevice(ctx->device));
  std::vector<uint8_t> tags((size_t)m);
  const int rc = lso::download_leaves(om->leaves, which, centres4, tags.data(), om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "leaf download failed");
  for (long long i = 0; i < m; ++i) {
    depths[i] = tags[i] & 31;
    states[i] = tags[i] & 32 ? LS_CELL_FREE : LS_CELL_OCCUPIED;
  }
  return LS_OK;
}

int ls_occupancy_marker_cubes(ls_occupancy* om, double min_z, double max_z, double color_factor, float* centres4,
                              float* colors4, int64_t occupied_offsets[18], int64_t free_offsets[18], int64_t cap, int64_t* n) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n) return fail(ctx, LS_ERR_ARG, "bad argument");
  *n = 0;
  if (cap < 0 || !occupied_offsets || !free_offsets || (cap > 0 && (!centres4 || !colors4)))
    return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!std::isfinite(min_z) || !std::isfinite(max_z) || !std::isfinite(color_factor) || !(min_z < max_z) ||
      !std::isfinite(max_z - min_z))
    return fail(ctx, LS_ERR_ARG, "colour arguments min_z %g, max_z %g, color_factor %g (finite, min_z < max_z)", min_z, max_z,
                color_factor);
  if (om->leaves_version != om->version)
    return fail(ctx, LS_ERR_STATE, "no current leaf list: build it after the last change to the map");
  const lso::Leaves& L = om->leaves;
  occupied_offsets[0] = 0;
  for (int d = 0; d < 17; ++d) occupied_offsets[d + 1] = occupied_offsets[d] + L.occupied[d];
  free_offsets[0] = occupied_offsets[17];
  for (int d = 0; d < 17; ++d) free_offsets[d + 1] = free_offsets[d] + L.free[d];
  *n = free_offsets[17];
  if (*n > cap) return fail(ctx, LS_ERR_ARG, "buffers of %lld cubes for %lld", (long long)cap, (long long)*n);
  CU(cudaSetDevice(ctx->device));
  const int rc = lso::marker_cubes(om->leaves, min_z, max_z, color_factor, centres4, colors4, om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "marker cubes failed");
  return LS_OK;
}

int ls_occupancy_build_projection(ls_occupancy* om, double min_z, double max_z, double min_size_x, double min_size_y,
                                  ls_grid_info* info) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!info) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (std::isnan(min_z) || std::isnan(max_z)) return fail(ctx, LS_ERR_ARG, "band min_z %g, max_z %g has a NaN", min_z, max_z);
  if (!std::isfinite(min_size_x) || !std::isfinite(min_size_y) || min_size_x < 0.0 || min_size_y < 0.0)
    return fail(ctx, LS_ERR_ARG, "minimum size %g x %g (finite, >= 0)", min_size_x, min_size_y);
  CU(cudaSetDevice(ctx->device));
  // The projection's version is not reset first: on a failure here or in the .bt build, the last projection stays as it
  // was, and current if it was.
  bool built;
  int rc = current_tree(om, TreeFormat::Binary, &built);
  if (rc) return rc;
  ls_occupancy::Tree& t = tree_of(om, TreeFormat::Binary);
  CU(om->clock.start());
  const char* why = "";
  rc = lso::build_projection(om->map, om->prm, t.tree, lso::ProjectionArgs{min_z, max_z, min_size_x, min_size_y},
                             om->projection, &why, om->clock.stream, &ctx->launches);
  if (rc == LS_ERR_ARG || (rc == LS_ERR_NOMEM && *why)) return fail(ctx, rc, "2D projection: %s", why);
  if (rc) return fail_lso(ctx, rc, "2D projection");
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  om->projection_version = om->version;
  const lso::Projection& p = om->projection;
  info->width = p.width, info->height = p.height;
  info->resolution = om->prm.res;
  info->origin_x = p.origin[0], info->origin_y = p.origin[1];
  info->unknown_cells = p.cells[0], info->free_cells = p.cells[1], info->occupied_cells = p.cells[2];
  info->device_ms = ms + (built ? t.ms : 0.f);
  return LS_OK;
}

int ls_occupancy_download_projection(ls_occupancy* om, int8_t* data, int64_t cap) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (om->projection_version != om->version)
    return fail(ctx, LS_ERR_STATE, "no current 2D projection: build it after the last change to the map");
  const lso::Projection& p = om->projection;
  const long long cells = p.width * p.height;
  if (cap < cells || (cells > 0 && !data))
    return fail(ctx, LS_ERR_ARG, "a buffer of %lld cells for %lld", (long long)cap, cells);
  CU(cudaSetDevice(ctx->device));
  const int rc = lso::download_projection(p, data, om->clock.stream);
  if (rc) return fail(ctx, rc, "2D projection download failed");
  return LS_OK;
}

int ls_occupancy_track_changes(ls_occupancy* om, int enable) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  CU(cudaSetDevice(ctx->device));
  if (!enable) {
    CU(cudaStreamSynchronize(om->clock.stream));
    lso::release_changes(om->changes);
    om->tracking = false;
    return LS_OK;
  }
  const int rc = lso::capture_baseline(om->changes, om->map, om->prm, om->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, rc == LS_ERR_NOMEM ? "change detection: out of device memory for the baseline" :
                                                    "change detection: baseline capture failed");
  om->tracking = true;
  return LS_OK;
}

int ls_occupancy_changes(ls_occupancy* om, uint64_t* keys, int8_t* status, int8_t* previous, float* centres4, int64_t cap,
                         int64_t* n, int reset, ls_occupancy_change_stats* stats) {
  if (!om) return LS_ERR_ARG;
  ls_ctx* ctx = om->ctx;
  if (!n) return fail(ctx, LS_ERR_ARG, "bad argument");
  *n = 0;
  if (cap < 0) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!om->tracking) return fail(ctx, LS_ERR_STATE, "change detection is off: enable it with ls_occupancy_track_changes");
  CU(cudaSetDevice(ctx->device));
  CU(om->clock.start());
  const long long compared = (long long)om->map.pool_n + om->changes.base.n;
  long long m = 0;
  int rc = lso::diff_changes(om->changes, om->map, om->prm, keys, status, previous, centres4, cap, &m, om->clock.stream,
                             &ctx->launches);
  *n = m;
  if (rc == LS_ERR_ARG) return fail(ctx, rc, "buffers of %lld changes for %lld", (long long)cap, m);
  if (rc) return fail_lso(ctx, rc, "changes");
  if (reset && (rc = lso::capture_baseline(om->changes, om->map, om->prm, om->clock.stream, &ctx->launches)))
    return fail(ctx, rc, rc == LS_ERR_NOMEM ? "changes copied, the reset is refused: out of device memory for the baseline"
                                            : "changes copied, the reset failed");
  float ms = 0.f;
  CU(om->clock.stop(&ms));
  if (stats) {
    stats->bricks_compared = compared;
    stats->changed = m;
    stats->baseline_bricks = om->changes.base.n;
    stats->device_bytes = (int64_t)lso::changes_bytes(om->changes);
    stats->device_ms = ms;
  }
  return LS_OK;
}

}  // extern "C"

// ---- Euclidean distance map of the occupancy map (DynamicEDTOctomap; kernels in ls_distance.cu) --------------------------
struct ls_distance_map {
  ls_ctx* ctx = nullptr;
  ls_distance_map_params prm{};
  DeviceClock clock;
  lso::DistanceField field;
  bool has_field = false;
  float max_dist = 0.f;  // getMaxDist of the field
};

namespace {
void distance_stats(const ls_distance_map* dm, float ms, ls_distance_map_stats* stats) {
  if (!stats) return;
  const lso::DistanceField& f = dm->field;
  for (int a = 0; a < 3; ++a) stats->min_key[a] = f.kmin[a], stats->size[a] = f.size[a];
  stats->cells = f.cells;
  stats->obstacles = f.obstacles;
  stats->resolution = f.res;
  stats->max_sqdist_cells = f.M;
  stats->max_dist = dm->max_dist;
  stats->device_bytes = (int64_t)lso::distance_bytes(f);
  stats->device_ms = ms;
}
}  // namespace

extern "C" {

int ls_distance_map_create(ls_ctx* ctx, const ls_distance_map_params* params, ls_distance_map** out) {
  if (!ctx || !out) return LS_ERR_ARG;
  *out = nullptr;
  if (!params) return fail(ctx, LS_ERR_ARG, "bad argument");
  const ls_distance_map_params& p = *params;
  if (!std::isfinite(p.max_dist) || !(p.max_dist > 0.f))
    return fail(ctx, LS_ERR_ARG, "distance map max_dist %g (finite and > 0)", (double)p.max_dist);
  for (int a = 0; a < 3; ++a) {
    if (!std::isfinite(p.bbx_min[a]) || !std::isfinite(p.bbx_max[a]))
      return fail(ctx, LS_ERR_ARG, "distance map box corner not finite on axis %d", a);
    if (p.bbx_min[a] > p.bbx_max[a])
      return fail(ctx, LS_ERR_ARG, "distance map box min %g > max %g on axis %d", (double)p.bbx_min[a], (double)p.bbx_max[a], a);
  }
  CU(cudaSetDevice(ctx->device));
  ls_distance_map* dm = new ls_distance_map();
  dm->ctx = ctx;
  dm->prm = p;
  if (!dm->clock.create()) {
    ls_distance_map_destroy(dm);
    return fail(ctx, LS_ERR_NOMEM, "distance map creation failed");
  }
  *out = dm;
  return LS_OK;
}

void ls_distance_map_destroy(ls_distance_map* dm) {
  if (!dm) return;
  cudaSetDevice(dm->ctx->device);
  dm->clock.destroy();
  delete dm;
}

int ls_distance_map_update(ls_distance_map* dm, ls_occupancy* om, ls_distance_map_stats* stats) {
  if (!dm) return LS_ERR_ARG;
  ls_ctx* ctx = dm->ctx;
  if (!om) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (om->ctx->device != ctx->device)
    return fail(ctx, LS_ERR_ARG, "the occupancy map is on device %d, the distance map on device %d", om->ctx->device,
                ctx->device);
  const ls_distance_map_params& p = dm->prm;
  const double res = om->prm.res, inv = om->prm.inv;
  const double mf = (double)p.max_dist / res + 1.0;
  if (!(mf < 46341.0)) return fail(ctx, LS_ERR_ARG, "max_dist %g is more than 46340 cells of %g m", (double)p.max_dist, res);
  const int m = (int)mf;
  int kmin[3], kmax[3];
  long long cells = 1;
  for (int a = 0; a < 3; ++a) {
    if (!lso::key_of(inv, p.bbx_min[a], kmin[a]) || !lso::key_of(inv, p.bbx_max[a], kmax[a]))
      return fail(ctx, LS_ERR_ARG, "a box corner has no valid key on axis %d at resolution %g", a, res);
    if (kmin[a] > kmax[a]) return fail(ctx, LS_ERR_ARG, "box min key above max key on axis %d", a);
    cells *= kmax[a] - kmin[a] + 1;
  }
  if (cells > (1LL << 30)) return fail(ctx, LS_ERR_ARG, "the box has %lld cells (at most 2^30)", cells);
  CU(cudaSetDevice(ctx->device));
  lso::DistanceField& f = dm->field;
  dm->has_field = false;
  int rc = lso::distance_reserve(f, cells);
  if (rc) return fail(ctx, rc, "distance map: out of device memory for %lld cells", cells);
  for (int a = 0; a < 3; ++a) f.kmin[a] = kmin[a], f.size[a] = kmax[a] - kmin[a] + 1;
  f.cells = cells;
  f.res = res, f.inv = inv;
  f.M = m * m;
  dm->max_dist = (float)(m * res);
  CU(dm->clock.start());
  rc = lso::distance_update(f, om->map, om->prm.l_occ, p.treat_unknown_as_occupied != 0, dm->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "distance map update failed");
  float ms = 0.f;
  CU(dm->clock.stop(&ms));
  dm->has_field = true;
  distance_stats(dm, ms, stats);
  return LS_OK;
}

int ls_distance_map_query(ls_distance_map* dm, const float* points3, int n, float* distance, int32_t* sqdist_cells,
                          float* obstacles3, ls_distance_map_query_stats* stats) {
  if (!dm) return LS_ERR_ARG;
  ls_ctx* ctx = dm->ctx;
  if (n < 0 || (n > 0 && !points3)) return fail(ctx, LS_ERR_ARG, "bad argument");
  if (!dm->has_field) return fail(ctx, LS_ERR_STATE, "the distance map has no field: update it first");
  CU(cudaSetDevice(ctx->device));
  CU(dm->clock.start());
  long long outside = 0;
  const int rc = lso::distance_query(dm->field, points3, n, distance, sqdist_cells, obstacles3, &outside, dm->clock.stream,
                                     &ctx->launches);
  if (rc) return fail_lso(ctx, rc, "distance query");
  float ms = 0.f;
  CU(dm->clock.stop(&ms));
  if (stats) {
    stats->outside = outside;
    stats->device_ms = ms;
  }
  return LS_OK;
}

int ls_distance_map_download(ls_distance_map* dm, int32_t* sqdist, uint64_t* obstacle_keys, int64_t cap_cells, int64_t* n) {
  if (!dm) return LS_ERR_ARG;
  ls_ctx* ctx = dm->ctx;
  if (!n) return fail(ctx, LS_ERR_ARG, "bad argument");
  *n = 0;
  if (!dm->has_field) return fail(ctx, LS_ERR_STATE, "the distance map has no field: update it first");
  *n = dm->field.cells;
  if (cap_cells < dm->field.cells)
    return fail(ctx, LS_ERR_ARG, "buffers of %lld cells for %lld", (long long)cap_cells, dm->field.cells);
  CU(cudaSetDevice(ctx->device));
  const int rc = lso::distance_download(dm->field, sqdist, obstacle_keys, dm->clock.stream, &ctx->launches);
  if (rc) return fail(ctx, rc, "distance map download failed");
  return LS_OK;
}

}  // extern "C"
