// Host orchestration + C ABI (include/rootba_b200.h) of the H100-native square-root BA inner loop.
// One rba_handle = one landmark shard on one GPU; everything is enqueued on one CUDA stream.
// "ref:" citations are relative to src/rootba/ of the reference (NikolausDemmel/rootba @ d3900037).
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "../../include/rootba_b200.h"
#include "../host/bal_io_fast.hpp"
#include "kernels.cuh"
#include "covariance.cuh"
#include "assembled.cuh"
#include "nccl_dyn.hpp"

namespace rba {

thread_local std::string g_err;

// the host builds the pair lists as IntPair (layout.hpp); the kernels read them as int2
static_assert(sizeof(IntPair) == sizeof(int2), "IntPair must have the layout of int2");

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess) {                                                                      \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e__) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"; \
      return RBA_ERR_CUDA;                                                                         \
    }                                                                                              \
  } while (0)
#define TRY(x) do { int rc_ = (x); if (rc_) return rc_; } while (0)

struct EventPair {
  cudaEvent_t a = nullptr, b = nullptr;
  bool used = false;
};

}  // namespace rba

using namespace rba;

// type-erased base so the C ABI can hold either scalar type
struct rba_handle {
  int scalar_size = 0;
  virtual ~rba_handle() {}
  virtual int set_state(const void* cams, const void* lms) = 0;
  virtual int get_state(void* cams, void* lms) = 0;
  virtual int backup() = 0;
  virtual int restore() = 0;
  virtual int set_camera_fixed(const uint8_t* flags) = 0;
  virtual int set_camera_prior(const void* mean, const void* sqrt_info) = 0;
  virtual int set_camera_pair_prior(int32_t num_pairs, const int32_t* pairs, const void* mean, const void* sqrt_info) = 0;
  virtual int set_landmark_prior(int32_t num, const int32_t* lm_idx, const void* mean, const void* sqrt_info) = 0;
  virtual int compute_error(rba_residual_info* out) = 0;
  virtual int linearize() = 0;
  virtual int solve(double lambda, void* inc_out, rba_cg_summary* cg) = 0;
  virtual int apply(const void* inc, void* l_diff_out, bool update_cameras) = 0;
  virtual int lm_step(bool linearize_first, double lambda, rba_lm_step_result* out) = 0;
  virtual int lm_run(const rba_lm_opts* o, int max_steps, rba_lm_iteration* log, int* steps_done, int* terminated, rba_stage_timings* totals) = 0;
  virtual int get_timings(rba_stage_timings* out) const = 0;
  virtual int get_stats(rba_workload_stats* out) const = 0;
  virtual int get_scaling(void* scaling, void* diag2) = 0;
  virtual int get_rhs(void* b) = 0;
  virtual int get_precond(void* inv, void* blocks) = 0;
  virtual int right_multiply(const void* x, void* y) = 0;
  virtual int debug_get_block(int lm, void* out, int rows, int cols, void* jls) = 0;
  virtual int compute_covariance(double* cam_cov, double* lm_cov) = 0;
  virtual int time_matvec(int reps, double* sec) = 0;
  virtual int timer_start() = 0;
  virtual int timer_stop(double* sec) = 0;
  virtual void* stream_ptr() = 0;
  virtual int synchronize() = 0;
  virtual int comm_init(const void* uid) = 0;
  virtual int ipc_export(void* out128) = 0;
  virtual int ipc_import(const void* all) = 0;
};

namespace rba {

template <class S>
struct Solver : rba_handle {
  static constexpr int EBLOCKS = 592;
  static constexpr int KPMAX = sizeof(S) == 4 ? 16 : 10;
  // tile kernels (linearize+QR, stage 2, panel gradient)
  static constexpr int TILE_WARPS = 4;
  static constexpr int K1_CAP = 3904;   // scalars of shared memory per warp: linearize+QR needs 60 * W * n + 64 (= 3904 for the standard tiles)
  static constexpr int K2_CAP = 3072;   // stage 2 needs 3 * W * CS + 9 * W * n + 20 W + 8 (<= 3048 for the standard tiles)
  // dense operator (k_matvec_small_tma, k_matvec_large)
  static constexpr int K4_WARPS = 4;
  static constexpr int K4_NS = 2;        // TMA ring stages per warp
  static constexpr int K4_STAGE = 4608;  // bytes per stage (2 rows of an f32 KP=9 tile)
  static constexpr size_t K4_SMEM_TMA = (size_t)K4_WARPS * K4_NS * K4_STAGE;
  // longest-first dealing of the small matvec items: cost = rows x KP (x 256 B) + this per-item constant (~12 KB-equivalent);
  // 0 / 16 / 48 / 128 measured within 1 % of each other
  static constexpr long long K4_ITEM_COST = 48;
  // streamed implicit operator: warps per block, slots per stage, stages per warp
  static constexpr int IMP_WARPS = 2, IMP_MAXSLOTS = 64, IMP_NS = 1;

  rba_solver_opts opt{};
  KOpts ko{};
  Layout L;
  int nc = 0, nl_total = 0;
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  size_t device_bytes = 0;
  DevPtrs<S> D{};
  // device-only helpers
  S* cams_bk = nullptr; S* lms_bk = nullptr;
  long long state_version = 0;     // bumped whenever cameras / landmarks change (set_state, apply, restore)
  rba_residual_info error_cache{}; long long error_cache_version = -1, error_enqueue_version = -1; bool error_cache_valid = false;
  bool error_enqueued = false;
  int* d_csr_obs_slots = nullptr; ReduceItem* d_csr_obs_items = nullptr; int* d_csr_obs_item_ptr = nullptr;
  int* d_csr_y_slots = nullptr; ReduceItem* d_csr_y_items = nullptr; int* d_csr_y_item_ptr = nullptr;
  int n_obs_items = 0, n_y_items = 0;
  // camera-major CSR the operator's per-slot output is reduced over: the y-slot CSR of the dense form (one slot per
  // observation and row chunk) or the observation CSR of the implicit form
  const int* op_slots = nullptr; const ReduceItem* op_items = nullptr; const int* op_item_ptr = nullptr; int n_op_items = 0;
  bool implicit_op = false;
  bool panel_form = true;        // gradient and SCHUR_JACOBI blocks from the Q2 panels (reference form) instead of the identities
  ReduceItem* d_pb_items = nullptr; int* d_pb_item_ptr = nullptr; int n_pb_items = 0;
  // launch geometry and work orders of the persistent kernels (deal_work, setup_kernels)
  Scratch<S> k1_sc{}, k2_sc{};
  size_t k1_smem = 0, k2_smem = 0;
  int k1_max_blocks = 264, k2_max_blocks = 264;
  TileOrder order_k1{nullptr, 0}, order_kp{nullptr, 0};
  MatvecItem* d_items = nullptr;   // L.items, the small-KP part dealt to the persistent warps of the TMA matvec
  int n_dealt = 0, tma_grid = 1;
  size_t k4_smem_small = 0;
  int imp_tile_split = 0;        // tiles [0, split) have <= IMP_MAXSLOTS slots and take the streamed kernel
  size_t imp_smem = 0; int imp_grid = 1;
  int pcg_cluster = 16;
  // test hooks (read_test_hooks)
  bool pcg_partials = true;      // one GPU: k_pcg_vec consumes the per-segment sums of k_cam_reduce
  bool peer_ar = true;           // rba_ipc_import maps the peers' exchange regions
  bool asm_hook = true;          // the assembled operator when it qualifies (setup_assembled)
  int asm_at = 0;                // > 0: build S at this PCG iteration instead of the break-even one
  int* h_prog = nullptr; int* d_prog = nullptr;  // PCG progress in host-mapped pinned memory: [0] last completed iteration, [1] solve ended
  int pcg_solve_id = 0;
  double* d_epart = nullptr;     // [EBLOCKS][6]
  double* d_red = nullptr;       // [8] reduced doubles (error / l_diff)
  int* d_flags = nullptr;        // [4] bad flags: [0] numerical failure, [1] peer-exchange time-out
  int* d_cam_cnt = nullptr;      // per-camera arrival counters of k_cam_reduce_final (zero between launches)
  PcgState* d_state = nullptr;
  PcgState* h_state = nullptr;   // pinned [2]
  // Pinned copies of d_red / d_flags, one slot per entry point, so that rba_lm_step can enqueue all of them and
  // synchronise once
  struct PinnedResults {
    double error[6];             // compute_error
    int error_flags[4];
    int linearize_flags[4];      // linearize
    double l_diff;               // apply
    int apply_flags[4];
  };
  PinnedResults* h_res = nullptr;
  cudaEvent_t poll_ev[2] = {nullptr, nullptr};
  // status
  bool linearized = false;
  bool new_linearization_point = false;
  bool have_inc = false;
  S last_lambda = 0;
  bool damping_valid = false;
  uint8_t* d_cam_fixed = nullptr;  // [nc] flags of rba_set_camera_fixed; D.cam_fixed points here while any flag is set
  bool all_cams_fixed = false;     // no free camera parameter: the reduced system is empty and its solve is skipped
  // camera priors (rba_set_camera_prior, DESIGN.md section 14); has_abs_prior while any L_c is non-zero.  D.prior_H points at
  // d_prior_H while there are absolute or pair priors.
  bool has_abs_prior = false;
  S* d_prior_mean = nullptr;       // [nc][10] mean, quaternion normalised
  S* d_prior_L = nullptr;          // [nc][81] square-root information
  S* d_prior_A = nullptr;          // [nc][81] L de/d(inc): unscaled after k_prior_linearize, scaled after k_prior_scale
  S* d_prior_r = nullptr;          // [nc][9]  L e at the linearisation point
  S* d_prior_H = nullptr;          // [nc][81] A^T A (+ the pair priors' diagonal blocks)
  S* d_prior_g = nullptr;          // [nc][9]  A^T r (+ the pair priors' A_s^T r)
  // pair priors (rba_set_camera_pair_prior, DESIGN.md section 15): n_pairs pairs with a non-zero L, D.pair_ov set while
  // n_pairs > 0.  Buffers are sized for pair_cap pairs.
  int n_pairs = 0, pair_cap = 0;
  int* d_pair_ij = nullptr;        // [m][2] cameras (i, j)
  S* d_pair_mean = nullptr;        // [m][7] R0 quaternion (normalised), t0
  S* d_pair_L = nullptr;           // [m][36] square-root information
  S* d_pair_A = nullptr;           // [m][2][36] pose blocks A_i, A_j: unscaled after k_pair_linearize, scaled after k_pair_scale
  S* d_pair_r = nullptr;           // [m][6] L e at the linearisation point
  int* d_pair_item = nullptr;      // [2m] incident sides 2 p + side, camera-major (CSR d_pair_ptr)
  int* d_pair_nbr = nullptr;       // [2m] the other camera of each side
  S* d_pair_O = nullptr;           // [2m][36] O of each directed edge
  int* d_pair_ptr = nullptr;       // [nc + 1]
  S* d_pair_ov = nullptr;          // [9 nc]
  // landmark priors (rba_set_landmark_prior, DESIGN.md section 17): the n_lmp priors of this shard with a non-zero L;
  // D.lmp_slot set while n_lmp > 0.  Buffers are sized for lmp_cap priors.
  int n_lmp = 0, lmp_cap = 0;
  int* d_lmp_slot = nullptr;       // [nsorted] prior slot per sorted landmark, -1 = none
  int* d_lmp_of_lm = nullptr;      // [nl_local] prior slot per local landmark, -1 = none (rba_compute_covariance)
  int* d_lmp_lm = nullptr;         // [m] local landmark of each prior
  S* d_lmp_mean = nullptr;         // [m][3]
  S* d_lmp_L = nullptr;            // [m][9]
  S* d_lmp_Lg = nullptr;           // [m][12]
  rba_stage_timings tm{};
  EventPair ev_stage1, ev_stage2, ev_precond, ev_pcg, ev_backsub, ev_update, ev_error, ev_mv, ev_user;
  long long launches = 0;
  long long lin_l0 = 0, solve_l0 = 0, apply_l0 = 0;  // `launches` at the start of the last linearize / solve / apply
  // NCCL
  NcclApi* nccl = nullptr;
  ncclComm_t comm = nullptr;
  // peer-memory all-reduce fused into the PCG vector kernel
  char* peer_mem = nullptr;      // this rank's exchange region (flags + staging areas, see PeerComm), IPC-exported
  size_t peer_bytes = 0;
  PeerComm pc{};
  bool peer_ok = false;
  int ar_seq = 0, c_seq = 0, s_seq = 0;  // sequence numbers of the three flag families (operator output / vectors / scalars)
  std::vector<void*> ipc_opened;
  // rba_compute_covariance (DESIGN.md section 16): the co-visible camera pairs and their (slot_a, slot_b) terms, and each
  // landmark's first slot and track length, built at the first call
  bool cov_ready = false;
  int cov_nblk = 0;
  IntPair* d_cov_blk_cam = nullptr; int* d_cov_blk_ptr = nullptr; IntPair* d_cov_terms = nullptr;
  int* d_cov_lm_slot0 = nullptr; int* d_cov_lm_n = nullptr;
  // assembled operator (setup_assembled, assembled.cuh): the terms as panel addresses in landmark-major order, the pair
  // list (term ranges, landmark-major position of every term), per pair its positions (lower, upper or -1) in the full
  // block-row CSR of S, the staging buffer of all terms, S_u per pair and S
  // asm_on: the structure exists; su_valid: S_u belongs to the current linearisation; s_valid: S = S_u + the damping part of
  // the last solve's lambda, and that solve (and rba_right_multiply / rba_time_matvec after it) applies S
  bool asm_on = false, su_valid = false, s_valid = false;
  int asm_nblk = 0, asm_switch = 0; long long asm_nt = 0, asm_nnzb = 0;
  AsmTerm* d_asm_terms = nullptr; int* d_asm_wpos = nullptr; int* d_asm_blk_ptr = nullptr; IntPair* d_asm_pos = nullptr;
  int* d_asm_row_ptr = nullptr; int* d_asm_col = nullptr;
  S* d_asm_stage = nullptr; S* d_asm_Su = nullptr; S* d_asm_S = nullptr;

  ~Solver() override {
    if (comm && nccl) nccl->CommDestroy(comm);
    for (void* p : ipc_opened) cudaIpcCloseMemHandle(p);
    for (void* p : allocs) cudaFree(p);
    if (h_prog) cudaFreeHost(h_prog);
    if (h_state) cudaFreeHost(h_state);
    if (h_res) cudaFreeHost(h_res);
    for (EventPair* e : {&ev_stage1, &ev_stage2, &ev_precond, &ev_pcg, &ev_backsub, &ev_update, &ev_error, &ev_mv, &ev_user}) {
      if (e->a) cudaEventDestroy(e->a);
      if (e->b) cudaEventDestroy(e->b);
    }
    for (auto& e : poll_ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }

  template <class T>
  int dalloc(T** p, size_t count, bool zero = true) {
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    void* q = nullptr;
    CU(cudaMalloc(&q, bytes));
    allocs.push_back(q);
    device_bytes += bytes;
    if (zero) CU(cudaMemsetAsync(q, 0, bytes, stream));
    *p = (T*)q;
    return RBA_OK;
  }
  // frees a buffer of dalloc (nullptr: nothing to do); device_bytes keeps counting it (the most the handle has allocated)
  int dfree(void* q) {
    if (!q) return RBA_OK;
    allocs.erase(std::find(allocs.begin(), allocs.end(), q));
    CU(cudaFree(q));
    return RBA_OK;
  }
  template <class T>
  int upload(T** p, const std::vector<T>& v) {
    int rc = dalloc(p, v.size(), false);
    if (rc) return rc;
    if (!v.empty()) CU(cudaMemcpyAsync(*p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream));
    return RBA_OK;
  }

  int start(EventPair& e) { e.used = true; CU(cudaEventRecord(e.a, stream)); return RBA_OK; }
  int stop(EventPair& e) { CU(cudaEventRecord(e.b, stream)); return RBA_OK; }
  static double elapsed(EventPair& e) {
    if (!e.used) return 0.0;
    float ms = 0;
    if (cudaEventElapsedTime(&ms, e.a, e.b) != cudaSuccess) return 0.0;
    return 1e-3 * ms;
  }

  // ------------------------------------------------------------------------------------------
  // Set-up, in this order: the options, the layout, the dealing of the work to the persistent kernels, the device buffers,
  // the tile scratch and the kernel attributes.
  int init(const rba_problem_view* pv, const rba_solver_opts* o) {
    TRY(validate_options(*o));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
      g_err = "no CUDA device: rootba_b200 has no CPU fallback";
      return RBA_ERR_NO_DEVICE;
    }
    if (opt.device >= 0) CU(cudaSetDevice(opt.device));
    CU(cudaGetDevice(&device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    sm_count = prop.multiProcessorCount;
    CU(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (EventPair* e : {&ev_stage1, &ev_stage2, &ev_precond, &ev_pcg, &ev_backsub, &ev_update, &ev_error, &ev_mv, &ev_user}) {
      CU(cudaEventCreate(&e->a));
      CU(cudaEventCreate(&e->b));
    }
    for (auto& e : poll_ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    read_test_hooks();
    TRY(upload_layout(pv));
    TRY(deal_work());
    TRY(alloc_buffers());
    TRY(setup_assembled());
    TRY(setup_kernels());
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }

  int validate_options(const rba_solver_opts& o) {
    opt = o;
    if (opt.nranks < 1 || opt.rank < 0 || opt.rank >= opt.nranks) { g_err = "bad rank/nranks"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.operator_form != 0 && opt.operator_form != 1) { g_err = "operator_form must be 0 (dense) or 1 (implicit)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.solver_type < 0 || opt.solver_type > 2) { g_err = "solver_type must be 0 (SQUARE_ROOT), 1 (SCHUR_COMPLEMENT) or 2 (POWER_SCHUR_COMPLEMENT)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.solver_type == 2 && opt.nranks > 1) { g_err = "POWER_SCHUR_COMPLEMENT runs on one GPU (the power-series vector kernel has no peer exchange yet)"; return RBA_ERR_UNSUPPORTED; }
    if (opt.stage2_form != 0 && opt.stage2_form != 1) { g_err = "stage2_form must be 0 (Q2 panel, reference) or 1 (orthogonality identity)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.pcg_check_period <= 0) opt.pcg_check_period = 4;
    if (opt.residual_reset_period <= 0) opt.residual_reset_period = 10;
    if (opt.power_order <= 0) opt.power_order = 20;  // solver_options.hpp:270
    // the Schur-complement solvers share the per-observation records and the implicit operator kernels (k_sc_stage2)
    implicit_op = opt.operator_form == 1 || opt.solver_type != 0;
    // gradient / SCHUR_JACOBI blocks from the stored Q2 panels like the reference, unless there are no panels (implicit operator)
    panel_form = !implicit_op && opt.stage2_form == 0;
    ko.use_valid_projections_only = opt.use_valid_projections_only;
    ko.robust_norm = opt.robust_norm;
    ko.write_panel = implicit_op ? 0 : 1;
    ko.huber = opt.huber_parameter;
    ko.jacobi_eps = opt.jacobi_scaling_epsilon > 0 ? opt.jacobi_scaling_epsilon : (double)ST<S>::eps_sqrt();  // ref: linearizor_base.cpp:72-79
    return RBA_OK;
  }

  // Test hooks, not options: each forces at small size a path that the solver also takes on its own.
  //   RBA_PCG_PARTIALS=0  PCG without the per-segment hand-over to the vector kernel (taken above 1808 cameras)
  //   RBA_PCG_CLUSTER=k   a PCG vector cluster of at most k CTAs (taken when the device grants fewer than 16)
  //   RBA_PEER_AR=0       NCCL for the reductions across shards (taken when the IPC mapping of a peer fails)
  //   RBA_ASSEMBLED_RCS=0 the panel product P^T (P x) instead of the assembled S x (taken when S does not qualify)
  //   RBA_ASSEMBLED_AT=k  S built at PCG iteration k instead of the break-even iteration (taken by solves that run long)
  void read_test_hooks() {
    if (const char* e = getenv("RBA_PCG_PARTIALS")) pcg_partials = atoi(e) != 0;
    if (const char* e = getenv("RBA_PCG_CLUSTER")) pcg_cluster = std::max(1, std::min(atoi(e), 16));
    if (const char* e = getenv("RBA_PEER_AR")) peer_ar = atoi(e) != 0;
    if (const char* e = getenv("RBA_ASSEMBLED_RCS")) asm_hook = atoi(e) != 0;
    if (const char* e = getenv("RBA_ASSEMBLED_AT")) asm_at = std::max(0, atoi(e));
  }

  int upload_layout(const rba_problem_view* pv) {
    nc = pv->num_cameras;
    nl_total = pv->num_landmarks;
    std::string msg = build_layout(nc, nl_total, pv->lm_obs_offset, pv->obs_cam_idx, opt.rank, opt.nranks, KPMAX, L);
    if (!msg.empty()) { g_err = msg; return RBA_ERR_INVALID_ARGUMENT; }
    // observation coordinates in slot order
    std::vector<S> xy((size_t)2 * L.nslots, S(0));
    const S* src = (const S*)pv->obs_xy;
    for (int s = 0; s < L.nslots; ++s)
      if (L.slot_obs[s] >= 0) { xy[2 * (size_t)s] = src[2 * L.slot_obs[s]]; xy[2 * (size_t)s + 1] = src[2 * L.slot_obs[s] + 1]; }
    TileInfo* d_tiles; int* d_sorted; int* d_slot_cam; int* d_slot_lm; S* d_xy;
    TRY(upload(&d_tiles, L.tiles));
    TRY(upload(&d_sorted, L.sorted_lm));
    TRY(upload(&d_slot_cam, L.slot_cam));
    TRY(upload(&d_slot_lm, L.slot_lm));
    TRY(upload(&d_xy, xy));
    D.tiles = d_tiles; D.ntiles = (int)L.tiles.size(); D.sorted_lm = d_sorted;
    D.slot_cam = d_slot_cam; D.slot_lm = d_slot_lm; D.slot_xy = d_xy; D.nslots = L.nslots; D.nc = nc;
    TRY(upload(&d_csr_obs_slots, L.csr_obs.slots));
    TRY(upload(&d_csr_obs_items, L.csr_obs.items));
    TRY(upload(&d_csr_obs_item_ptr, L.csr_obs.cam_item_ptr));
    n_obs_items = (int)L.csr_obs.items.size();
    if (L.csr_y_is_obs) {
      d_csr_y_slots = d_csr_obs_slots; d_csr_y_items = d_csr_obs_items; d_csr_y_item_ptr = d_csr_obs_item_ptr;
      n_y_items = n_obs_items;
    } else {
      TRY(upload(&d_csr_y_slots, L.csr_y.slots));
      TRY(upload(&d_csr_y_items, L.csr_y.items));
      TRY(upload(&d_csr_y_item_ptr, L.csr_y.cam_item_ptr));
      n_y_items = (int)L.csr_y.items.size();
    }
    if (implicit_op) { op_slots = d_csr_obs_slots; op_items = d_csr_obs_items; op_item_ptr = d_csr_obs_item_ptr; n_op_items = n_obs_items; }
    else { op_slots = d_csr_y_slots; op_items = d_csr_y_items; op_item_ptr = d_csr_y_item_ptr; n_op_items = n_y_items; }
    TRY(upload(&d_pb_items, L.pb_items));
    TRY(upload(&d_pb_item_ptr, L.pb_cam_item_ptr));
    n_pb_items = (int)L.pb_items.size();
    return RBA_OK;
  }

  // The grids of the persistent kernels and the order in which their warps take the work.
  int deal_work() {
    if (implicit_op) {
      while (imp_tile_split < (int)L.tiles.size() && (32 / L.tiles[imp_tile_split].G) * L.tiles[imp_tile_split].n <= IMP_MAXSLOTS) ++imp_tile_split;
      imp_smem = (size_t)IMP_WARPS * IMP_NS * (size_t)IMP_MAXSLOTS * 48 * sizeof(S);
      CU(cudaFuncSetAttribute((k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)imp_smem));
      int bps = 0;
      CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, (k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), IMP_WARPS * 32, imp_smem));
      imp_grid = std::max(1, std::min((imp_tile_split + IMP_WARPS - 1) / IMP_WARPS, sm_count * std::max(1, bps)));
    } else {
      TRY(deal_matvec_items());
    }
    // the tile kernels' scratch decides k_linearize_qr's grid
    long long need1 = 0, need2 = 0;
    for (const TileInfo& T : L.tiles) {
      const int Wn = (32 / T.G) * T.n;
      need1 = std::max<long long>(need1, (long long)Wn * 60 + 64);
      need2 = std::max<long long>(need2, (long long)stage2_need(T.n, T.G, T.KP));
    }
    tile_scratch_geometry(k1_sc, K1_CAP, need1, k1_smem, k1_max_blocks);
    tile_scratch_geometry(k2_sc, K2_CAP, need2, k2_smem, k2_max_blocks);
    // tiles dealt to the persistent warps longest-first (the kernels' work per tile grows like n^2: panel rows x columns)
    TRY(deal_tiles(tile_grid(k1_max_blocks) * TILE_WARPS, order_k1));
    TRY(deal_tiles(tile_grid(sm_count * 8) * TILE_WARPS, order_kp));
    return RBA_OK;
  }

  // The persistent warps of the TMA matvec take the items q = first + k * (number of warps).  Dealing the items sorted by
  // size round-robin leaves a warp with up to 1.6x the mean work on Ladybug-1723 (13 045 items for 2 960 warps: some get 5,
  // some 4, and warp 0 the largest of every round); instead the small-KP items are dealt longest-processing-time-first
  // (deal_lpt), padded with empty items (nrows = 0 = end of a warp's list).  The grid must be exactly the co-resident CTAs
  // (shared memory: 5 per SM; the float64 instance is register-limited to 2), or the longest-first lists of a later wave
  // would start when the first is done.
  int deal_matvec_items() {
    CU(cudaFuncSetAttribute((k_matvec_small_tma<S, K4_WARPS, K4_NS, K4_STAGE>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K4_SMEM_TMA));
    int occ = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (k_matvec_small_tma<S, K4_WARPS, K4_NS, K4_STAGE>), K4_WARPS * 32, K4_SMEM_TMA));
    int bps = std::max(1, (int)((220 * 1024) / (K4_SMEM_TMA + 1024)));
    if (occ > 0) bps = std::min(bps, occ);
    const int nsmall = (int)L.items.size() - L.n_items_large;
    tma_grid = grid_for(nsmall, K4_WARPS, bps);
    const int W = tma_grid * K4_WARPS;
    std::vector<MatvecItem> items = L.items;
    if (nsmall > W) {
      std::vector<long long> cost(nsmall);
      for (int q = 0; q < nsmall; ++q) {
        const MatvecItem& it = L.items[L.n_items_large + q];
        cost[q] = (long long)it.nrows * L.tiles[it.tile].KP + K4_ITEM_COST;
      }
      const MatvecItem empty{};
      items.resize(L.n_items_large);
      for (int q : deal_lpt(cost, W)) items.push_back(q >= 0 ? L.items[L.n_items_large + q] : empty);
    }
    n_dealt = (int)items.size();
    return upload(&d_items, items);
  }

  // longest-first tile order for nw persistent warps of the tile kernels (none when every warp gets at most one tile)
  int deal_tiles(int nw, TileOrder& out) {
    const int nt = (int)L.tiles.size();
    if (nt <= nw) return RBA_OK;
    std::vector<long long> cost(nt);
    for (int t = 0; t < nt; ++t) {
      const TileInfo& T = L.tiles[t];
      cost[t] = (long long)2 * T.n * T.KP + (long long)(32 / T.G) * T.n / 2 + 8;  // panel rows x column steps + per-observation work + constant
    }
    int* d = nullptr;
    const std::vector<int> order = deal_lpt(cost, nw);
    TRY(upload(&d, order));
    out.order = d; out.count = (int)order.size();
    return RBA_OK;
  }

  // tile kernels (linearize+QR, stage 2): scratch in shared memory when the tile fits in the kernel's cap (scalars per
  // warp), else in a per-warp slice of a global buffer of at most 1 GiB (very long tracks; slow but general), which
  // limits the grid
  void tile_scratch_geometry(Scratch<S>& sc, int cap, long long need, size_t& smem, int& max_blocks) const {
    sc.smem_cap = cap; sc.gbase = nullptr; sc.gstride = 0;
    smem = (size_t)TILE_WARPS * cap * sizeof(S);
    max_blocks = sm_count * std::max(1, (int)((220 * 1024) / (smem + 1024)));
    if (need > cap) {
      long long warps = (long long)max_blocks * TILE_WARPS;
      while (warps > TILE_WARPS && warps * need * (long long)sizeof(S) > (1LL << 30)) warps /= 2;
      max_blocks = (int)std::max<long long>(1, warps / TILE_WARPS);
      sc.gstride = (need + 3) & ~3LL;
    }
  }

  int alloc_buffers() {
    TRY(dalloc(&D.cams, (size_t)10 * nc)); TRY(dalloc(&cams_bk, (size_t)10 * nc));
    TRY(dalloc(&D.lms, (size_t)3 * L.nl_local)); TRY(dalloc(&lms_bk, (size_t)3 * L.nl_local));
    if (ko.write_panel) TRY(dalloc(&D.panel, (size_t)L.panel_scalars));  // the implicit operator never touches the panels
    TRY(dalloc(&D.jp, (size_t)20 * L.nslots));
    TRY(dalloc(&D.q1u, (size_t)28 * L.nslots));
    TRY(dalloc(&D.q1d, (size_t)28 * L.nslots));
    TRY(dalloc(&D.jl, (size_t)6 * L.nslots));
    TRY(dalloc(&D.res, (size_t)2 * L.nslots));
    TRY(dalloc(&D.lmk, (size_t)24 * L.sorted_lm.size()));
    TRY(dalloc(&D.qtr, (size_t)2 * L.nslots));
    if (panel_form) {
      TRY(dalloc(&D.dmp, (size_t)28 * L.nslots));
      if (opt.preconditioner_type == 1) TRY(dalloc(&D.blk0, (size_t)48 * L.nslots));
      TRY(dalloc(&D.blocks0, (size_t)81 * nc));
      TRY(dalloc(&D.b0, (size_t)9 * nc));
    }
    for (S** v : {&D.diag2, &D.scaling, &D.b, &D.x, &D.r, &D.z, &D.p, &D.q, &D.y, &D.inc}) TRY(dalloc(v, (size_t)9 * nc));
    TRY(dalloc(&D.blocks, (size_t)81 * nc)); TRY(dalloc(&D.jblocks, (size_t)81 * nc)); TRY(dalloc(&D.inv, (size_t)81 * nc));
    TRY(dalloc(&D.yobs, (size_t)9 * L.nyslots));
    TRY(dalloc(&D.partial, (size_t)9 * std::max(n_obs_items, n_y_items)));
    TRY(dalloc(&D.pblk, (size_t)48 * n_pb_items));

    pc.nranks = 1; pc.rank = opt.rank;
    if (opt.nranks > 1 && opt.nranks <= MAX_PEERS) {
      pc.off_y = 4096;
      pc.off_c = pc.off_y + (((long long)2 * opt.nranks * 9 * nc * (long long)sizeof(S) + 255) & ~255LL);
      pc.cmax = (long long)81 * nc;
      peer_bytes = (size_t)(pc.off_c + (long long)2 * opt.nranks * pc.cmax * (long long)sizeof(S));
      TRY(dalloc(&peer_mem, peer_bytes));
      pc.base[opt.rank] = peer_mem;
      TRY(dalloc(&pc.dead, 1));
    }
    TRY(dalloc(&d_epart, (size_t)EBLOCKS * 6)); TRY(dalloc(&d_red, 8)); TRY(dalloc(&d_flags, 4));
    TRY(dalloc(&d_cam_cnt, (size_t)nc));
    TRY(dalloc(&d_state, 1));
    CU(cudaHostAlloc((void**)&h_prog, 64, cudaHostAllocMapped));
    CU(cudaHostGetDevicePointer((void**)&d_prog, h_prog, 0));
    h_prog[0] = 0; h_prog[1] = 0;
    CU(cudaMallocHost((void**)&h_state, 2 * sizeof(PcgState)));
    CU(cudaMallocHost((void**)&h_res, sizeof(PinnedResults)));
    return RBA_OK;
  }

  int setup_kernels() {
    if (k1_sc.gstride) TRY(dalloc(&k1_sc.gbase, (size_t)(k1_max_blocks * TILE_WARPS) * k1_sc.gstride, false));
    if (k2_sc.gstride) TRY(dalloc(&k2_sc.gbase, (size_t)(k2_max_blocks * TILE_WARPS) * k2_sc.gstride, false));
    CU(cudaFuncSetAttribute((k_linearize_qr<S, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CU(cudaFuncSetAttribute((k_linearize_qr<S, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
    // the landmark-prior instances (DESIGN.md section 17)
    CU(cudaFuncSetAttribute((k_linearize_qr<S, false, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CU(cudaFuncSetAttribute((k_linearize_qr<S, true, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, true, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, false, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
    k4_smem_small = (size_t)K4_WARPS * L.k4_scratch_per_warp * sizeof(S);
    if (k4_smem_small > 200 * 1024) { g_err = "matvec scratch exceeds shared memory"; return RBA_ERR_UNSUPPORTED; }
    CU(cudaFuncSetAttribute((k_matvec_large<S, K4_WARPS, KPMAX>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(k4_smem_small, 1024)));
    // the PCG vector step runs on one thread-block cluster (16 CTAs if the device grants it, else 8, ...)
    CU(cudaFuncSetAttribute(k_pcg_vec<S>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CU(cudaFuncSetAttribute((k_pcg_vec<S, true>), cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CU(cudaFuncSetAttribute((k_pcg_vec<S, true, true>), cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CU(cudaFuncSetAttribute(k_power_vec<S>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CU(cudaFuncSetAttribute((k_power_vec<S, true>), cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    for (; pcg_cluster > 1; pcg_cluster >>= 1) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(pcg_cluster); cfg.blockDim = dim3(VEC_THREADS);
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = pcg_cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int ncl = 0;
      if (cudaOccupancyMaxActiveClusters(&ncl, k_pcg_vec<S>, &cfg) == cudaSuccess && ncl >= 1) break;
      cudaGetLastError();
    }
    return RBA_OK;
  }

  // ------------------------------------------------------------------------------------------
  // sum over the shards, in place, on the solver stream: peer-memory push exchange when the ranks have mapped each other's
  // regions (rba_ipc_import), else NCCL
  int allreduce(S* buf, size_t count) {
    if (opt.nranks == 1) return RBA_OK;
    if (peer_ok && (long long)count <= pc.cmax) {
      ++c_seq;
      const int g = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm_count, (count + 255) / 256));
      k_peer_push<S><<<g, 256, 0, stream>>>(pc, buf, (long long)count, c_seq & 1);
      k_peer_sum<S><<<g, 256, 0, stream>>>(pc, buf, (long long)count, c_seq & 1, c_seq, d_flags + 1);
      launches += 2;
      return RBA_OK;
    }
    if (!comm) { g_err = "rba_comm_init has not been called on a sharded handle"; return RBA_ERR_STATE; }
    ncclResult_t r = nccl->AllReduce(buf, buf, count, sizeof(S) == 4 ? ncclFloat : ncclDouble, ncclSum, comm, stream);
    if (r != ncclSuccess) { g_err = std::string("ncclAllReduce: ") + nccl->GetErrorString(r); return RBA_ERR_NCCL; }
    return RBA_OK;
  }
  // nd doubles (d_red) and the bad flags (d_flags, summed = OR) in one exchange
  int allreduce_scalars(int nd) {
    if (opt.nranks == 1) return RBA_OK;
    if (peer_ok) {
      ++s_seq;
      k_peer_small<<<1, 64, 0, stream>>>(pc, d_red, nd, d_flags, 4, s_seq & 1, s_seq, d_flags + 1);
      ++launches;
      return RBA_OK;
    }
    if (!comm) { g_err = "rba_comm_init has not been called on a sharded handle"; return RBA_ERR_STATE; }
    ncclResult_t r = ncclSuccess;
    if (nd > 0) r = nccl->AllReduce(d_red, d_red, nd, ncclDouble, ncclSum, comm, stream);
    if (r == ncclSuccess) r = nccl->AllReduce(d_flags, d_flags, 4, ncclInt, ncclSum, comm, stream);
    if (r != ncclSuccess) { g_err = std::string("ncclAllReduce: ") + nccl->GetErrorString(r); return RBA_ERR_NCCL; }
    return RBA_OK;
  }

  int comm_init(const void* uid) override {
    if (opt.nranks == 1) return RBA_OK;
    nccl = nccl_api();
    if (!nccl) { g_err = "libnccl.so.2 could not be loaded"; return RBA_ERR_NCCL; }
    ncclUniqueId id;
    std::memcpy(&id, uid, sizeof(id));
    CU(cudaSetDevice(device));
    ncclResult_t r = nccl->CommInitRank(&comm, opt.nranks, id, opt.rank);
    if (r != ncclSuccess) { g_err = std::string("ncclCommInitRank: ") + nccl->GetErrorString(r); return RBA_ERR_NCCL; }
    return RBA_OK;
  }

  int ipc_export(void* out128) override {
    std::memset(out128, 0, 128);
    if (!peer_mem) return RBA_OK;  // single rank
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, peer_mem));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    std::memcpy(out128, &h, 64);
    return RBA_OK;
  }
  int ipc_import(const void* all) override {
    if (opt.nranks == 1) return RBA_OK;
    if (opt.nranks > MAX_PEERS) { g_err = "the peer-memory exchange supports at most 8 ranks"; return RBA_ERR_UNSUPPORTED; }
    if (!peer_ar) return RBA_OK;  // test hook (read_test_hooks): NCCL
    CU(cudaSetDevice(device));
    for (int r = 0; r < opt.nranks; ++r) {
      if (r == opt.rank) continue;
      cudaIpcMemHandle_t h;
      std::memcpy(&h, (const char*)all + (size_t)128 * r, 64);
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        g_err = "cudaIpcOpenMemHandle failed; using NCCL for the reductions across shards";
        return RBA_OK;  // peer_ok stays false: NCCL
      }
      ipc_opened.push_back(p);
      pc.base[r] = (char*)p;
    }
    pc.nranks = opt.nranks; pc.rank = opt.rank;
    peer_ok = true;
    return RBA_OK;
  }

  // ------------------------------------------------------------------------------------------
  int set_state(const void* cams, const void* lms) override {
    ++state_version;
    CU(cudaMemcpyAsync(D.cams, cams, (size_t)10 * nc * sizeof(S), cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(D.lms, (const S*)lms + (size_t)3 * L.lm_begin, (size_t)3 * L.nl_local * sizeof(S), cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  int get_state(void* cams, void* lms) override {
    CU(cudaMemcpyAsync(cams, D.cams, (size_t)10 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync((S*)lms + (size_t)3 * L.lm_begin, D.lms, (size_t)3 * L.nl_local * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  int backup() override {  // ref: bal/bal_problem.cpp:590-598
    CU(cudaMemcpyAsync(cams_bk, D.cams, (size_t)10 * nc * sizeof(S), cudaMemcpyDeviceToDevice, stream));
    CU(cudaMemcpyAsync(lms_bk, D.lms, (size_t)3 * L.nl_local * sizeof(S), cudaMemcpyDeviceToDevice, stream));
    return RBA_OK;
  }
  int restore() override {  // ref: bal/bal_problem.cpp:600-608
    ++state_version;
    CU(cudaMemcpyAsync(D.cams, cams_bk, (size_t)10 * nc * sizeof(S), cudaMemcpyDeviceToDevice, stream));
    CU(cudaMemcpyAsync(D.lms, lms_bk, (size_t)3 * L.nl_local * sizeof(S), cudaMemcpyDeviceToDevice, stream));
    return RBA_OK;
  }
  // Held parameters restrict the reduced camera system to its free rows and columns; the masking happens once per solve
  // in k_precond_invert (see there) and in the camera update.  No flag set = the unmodified path (D.cam_fixed == nullptr).
  int set_camera_fixed(const uint8_t* flags) override {
    bool any = false, all = flags != nullptr;
    if (flags)
      for (int c = 0; c < nc; ++c) {
        if (flags[c] & ~RBA_FIX_ALL) {
          g_err = "rba_set_camera_fixed: camera " + std::to_string(c) + " has flags " + std::to_string(flags[c]) + ", only bits 0..3 (RBA_FIX_ALL = 15) are defined";
          return RBA_ERR_INVALID_ARGUMENT;
        }
        any = any || flags[c] != 0;
        all = all && flags[c] == RBA_FIX_ALL;
      }
    if (any) {
      if (!d_cam_fixed) { int rc = dalloc(&d_cam_fixed, (size_t)nc, false); if (rc) return rc; }
      CU(cudaMemcpyAsync(d_cam_fixed, flags, (size_t)nc, cudaMemcpyHostToDevice, stream));
      CU(cudaStreamSynchronize(stream));
    }
    D.cam_fixed = any ? d_cam_fixed : nullptr;
    all_cams_fixed = all;
    have_inc = false;  // the device-resident increment was solved under the previous flags
    return RBA_OK;
  }
  // Gaussian priors on the camera parameters.  They are part of the linearisation (Jacobi scaling, A, r), so a change needs a
  // new rba_linearize; the device-resident increment and the cost cache are discarded.  No prior (both NULL, or every L_c
  // zero) = the unmodified path (D.prior_H == nullptr).
  int set_camera_prior(const void* mean_v, const void* sqrt_info_v) override {
    if ((mean_v == nullptr) != (sqrt_info_v == nullptr)) {
      g_err = "rba_set_camera_prior: mean and sqrt_info must both be given or both be NULL";
      return RBA_ERR_INVALID_ARGUMENT;
    }
    bool any = false;
    std::vector<S> mean, Lsq;
    if (mean_v) {
      const S* m = (const S*)mean_v;
      const S* Ls = (const S*)sqrt_info_v;
      mean.assign(m, m + (size_t)10 * nc);
      Lsq.assign(Ls, Ls + (size_t)81 * nc);
      for (int c = 0; c < nc; ++c) {
        bool nonzero;
        const std::string why = check_prior(m + 10 * (size_t)c, 10, Ls + 81 * (size_t)c, 81, nonzero, mean.data() + 10 * (size_t)c);
        if (!why.empty()) {
          g_err = "rba_set_camera_prior: camera " + std::to_string(c) + " " + why;
          return RBA_ERR_INVALID_ARGUMENT;
        }
        any = any || nonzero;
      }
    }
    if (any) {
      TRY(grow_upload(!d_prior_mean, dbuf(d_prior_mean, (size_t)10 * nc, &mean), dbuf(d_prior_L, (size_t)81 * nc, &Lsq),
                      dbuf(d_prior_A, (size_t)81 * nc), dbuf(d_prior_r, (size_t)9 * nc)));
      TRY(alloc_prior_diag());
      CU(cudaStreamSynchronize(stream));
    }
    has_abs_prior = any;
    return priors_changed();
  }
  // The checks of every prior setter on one prior, in this order: a finite mean (nm entries), a finite sqrt_info (nL
  // entries) and, for the two camera kinds (q given), a mean quaternion within 1e-3 of unit norm, written normalised to q.
  // Returns why the prior is rejected ("" = accepted); nonzero = L has a non-zero entry.
  static std::string check_prior(const S* m, int nm, const S* Ls, int nL, bool& nonzero, S* q = nullptr) {
    nonzero = false;
    for (int k = 0; k < nm; ++k)
      if (!std::isfinite((double)m[k])) return "has a non-finite mean";
    for (int k = 0; k < nL; ++k) {
      const double v = (double)Ls[k];
      if (!std::isfinite(v)) return "has a non-finite sqrt_info";
      nonzero = nonzero || v != 0.0;
    }
    if (q) {
      double n2 = 0;
      for (int k = 0; k < 4; ++k) n2 += (double)m[k] * (double)m[k];
      const double n = std::sqrt(n2);
      if (!(std::fabs(n - 1.0) <= 1e-3)) return "has a mean quaternion of norm " + std::to_string(n) + " (must be within 1e-3 of 1)";
      for (int k = 0; k < 4; ++k) q[k] = (S)((double)m[k] / n);
    }
    return "";
  }
  // One device buffer of a group: its entries when (re)allocated and, for an input, the host data copied into it.
  template <class T>
  struct DevBuf { T*& p; size_t count; const std::vector<T>* src; };
  template <class T>
  static DevBuf<T> dbuf(T*& p, size_t count, const std::vector<T>* src = nullptr) { return {p, count, src}; }
  // Reallocates every buffer of the group when `grow` (contents not kept), then queues the copies of the inputs on the stream.
  template <class... T>
  int grow_upload(bool grow, DevBuf<T>... b) {
    int rc = RBA_OK;
    if (grow) {
      ((rc = rc ? rc : dfree(b.p)), ...);
      ((rc = rc ? rc : dalloc(&b.p, b.count, false)), ...);
    }
    ((rc = rc ? rc : copy_in(b.p, b.src)), ...);
    return rc;
  }
  template <class T>
  int copy_in(T* dst, const std::vector<T>* src) {
    if (src) CU(cudaMemcpyAsync(dst, src->data(), src->size() * sizeof(T), cudaMemcpyHostToDevice, stream));
    return RBA_OK;
  }
  int alloc_prior_diag() { return grow_upload(!d_prior_H, dbuf(d_prior_H, (size_t)81 * nc), dbuf(d_prior_g, (size_t)9 * nc)); }
  CameraPrior<S> camera_prior() const { return {D.cams, d_prior_mean, d_prior_L, d_prior_A, d_prior_r}; }
  PairPrior<S> pair_prior() const { return {D.cams, d_pair_ij, d_pair_mean, d_pair_L, d_pair_A, d_pair_r}; }
  int priors_changed() {
    D.prior_H = (has_abs_prior || n_pairs > 0) ? d_prior_H : nullptr;
    D.pair_ov = n_pairs > 0 ? d_pair_ov : nullptr;
    linearized = false;  // the scaling, A and r of the last linearisation belong to the previous priors
    damping_valid = false;
    have_inc = false;
    error_cache_valid = false;
    return RBA_OK;
  }
  // Relative pose priors between pairs of cameras (DESIGN.md section 15).  Like the absolute priors they are part of the
  // linearisation.  Pairs with an all-zero L are dropped here; none left (num_pairs == 0 or every L zero) = the unmodified
  // path (D.pair_ov == nullptr).  Every check runs before anything changes, so a rejected call leaves the previous pairs.
  int set_camera_pair_prior(int32_t num_pairs, const int32_t* pairs, const void* mean_v, const void* sqrt_info_v) override {
    auto bad = [&](const std::string& what) { g_err = "rba_set_camera_pair_prior: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (num_pairs < 0) return bad("num_pairs must be >= 0, got " + std::to_string(num_pairs));
    if (num_pairs > 0 && (!pairs || !mean_v || !sqrt_info_v)) return bad("pairs, mean and sqrt_info must be given when num_pairs > 0");
    const S* m = (const S*)mean_v;
    const S* Ls = (const S*)sqrt_info_v;
    std::vector<int> ij;
    std::vector<S> mean, Lsq;
    for (int p = 0; p < num_pairs; ++p) {
      const int i = pairs[2 * p], j = pairs[2 * p + 1];
      const std::string tag = "pair " + std::to_string(p);
      if (i < 0 || i >= nc || j < 0 || j >= nc) return bad(tag + " has a camera index outside [0, " + std::to_string(nc) + ")");
      if (i == j) return bad(tag + " joins camera " + std::to_string(i) + " to itself");
      bool nonzero;
      S q[4];
      const std::string why = check_prior(m + 7 * (size_t)p, 7, Ls + 36 * (size_t)p, 36, nonzero, q);
      if (!why.empty()) return bad(tag + " " + why);
      if (!nonzero) continue;
      ij.push_back(i); ij.push_back(j);
      mean.insert(mean.end(), q, q + 4);
      mean.insert(mean.end(), m + 7 * (size_t)p + 4, m + 7 * (size_t)(p + 1));
      Lsq.insert(Lsq.end(), Ls + 36 * (size_t)p, Ls + 36 * (size_t)(p + 1));
    }
    const int np = (int)(ij.size() / 2);
    if (np > 0) {
      // camera-major list of the incident sides, ascending pair within a camera (the fixed summation order of the kernels)
      std::vector<int> ptr(nc + 1, 0), item(2 * (size_t)np), nbr(2 * (size_t)np);
      for (int k = 0; k < 2 * np; ++k) ++ptr[ij[k] + 1];
      for (int c = 0; c < nc; ++c) ptr[c + 1] += ptr[c];
      std::vector<int> fill(ptr.begin(), ptr.end() - 1);
      for (int k = 0; k < 2 * np; ++k) {
        const int q = fill[ij[k]]++;
        item[q] = k;            // 2 p + side
        nbr[q] = ij[k ^ 1];
      }
      TRY(grow_upload(np > pair_cap, dbuf(d_pair_ij, 2 * (size_t)np, &ij), dbuf(d_pair_mean, 7 * (size_t)np, &mean),
                      dbuf(d_pair_L, 36 * (size_t)np, &Lsq), dbuf(d_pair_A, 72 * (size_t)np), dbuf(d_pair_r, 6 * (size_t)np),
                      dbuf(d_pair_item, 2 * (size_t)np, &item), dbuf(d_pair_nbr, 2 * (size_t)np, &nbr), dbuf(d_pair_O, 72 * (size_t)np)));
      pair_cap = std::max(pair_cap, np);
      TRY(grow_upload(!d_pair_ptr, dbuf(d_pair_ptr, (size_t)nc + 1, &ptr), dbuf(d_pair_ov, 9 * (size_t)nc)));
      TRY(alloc_prior_diag());
      CU(cudaStreamSynchronize(stream));
    }
    n_pairs = np;
    D.pair_ptr = d_pair_ptr;
    D.pair_nbr = d_pair_nbr;
    D.pair_O = d_pair_O;
    return priors_changed();
  }

  // Gaussian priors on landmark positions (DESIGN.md section 17).  Part of the linearisation (Jacobi scaling, L~, g), like
  // the camera priors.  Every rank receives the full list and keeps the priors of its own landmark shard.  Priors with an
  // all-zero L are dropped; none left in this shard = the unmodified kernels (D.lmp_slot == nullptr).  Every check runs
  // before anything changes, so a rejected call leaves the previous priors.
  int set_landmark_prior(int32_t num, const int32_t* idx, const void* mean_v, const void* sqrt_info_v) override {
    auto bad = [&](const std::string& what) { g_err = "rba_set_landmark_prior: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (num < 0) return bad("num must be >= 0, got " + std::to_string(num));
    if (num > 0 && (!idx || !mean_v || !sqrt_info_v)) return bad("lm_idx, mean and sqrt_info must be given when num > 0");
    const S* m = (const S*)mean_v;
    const S* Ls = (const S*)sqrt_info_v;
    std::vector<uint8_t> seen((size_t)nl_total, 0);
    std::vector<int> slot(L.sorted_lm.size(), -1), of_lm((size_t)L.nl_local, -1), lm;
    std::vector<S> mean, Lsq;
    for (int p = 0; p < num; ++p) {
      const int l = idx[p];
      const std::string tag = "prior " + std::to_string(p);
      if (l < 0 || l >= nl_total) return bad(tag + " has a landmark index outside [0, " + std::to_string(nl_total) + ")");
      if (seen[l]) return bad(tag + " repeats landmark " + std::to_string(l));
      seen[l] = 1;
      bool nonzero;
      const std::string why = check_prior(m + 3 * (size_t)p, 3, Ls + 9 * (size_t)p, 9, nonzero);
      if (!why.empty()) return bad(tag + " " + why);
      if (!nonzero || l < L.lm_begin || l >= L.lm_end) continue;
      const int q = (int)lm.size();
      lm.push_back(l - L.lm_begin);
      slot[L.sorted_of_lm[l - L.lm_begin]] = q;
      of_lm[l - L.lm_begin] = q;
      mean.insert(mean.end(), m + 3 * (size_t)p, m + 3 * (size_t)(p + 1));
      Lsq.insert(Lsq.end(), Ls + 9 * (size_t)p, Ls + 9 * (size_t)(p + 1));
    }
    const int np = (int)lm.size();
    if (np > 0) {
      TRY(grow_upload(np > lmp_cap, dbuf(d_lmp_lm, (size_t)np, &lm), dbuf(d_lmp_mean, 3 * (size_t)np, &mean),
                      dbuf(d_lmp_L, 9 * (size_t)np, &Lsq), dbuf(d_lmp_Lg, 12 * (size_t)np)));
      lmp_cap = std::max(lmp_cap, np);
      TRY(grow_upload(!d_lmp_slot, dbuf(d_lmp_slot, slot.size(), &slot), dbuf(d_lmp_of_lm, of_lm.size(), &of_lm)));
      CU(cudaStreamSynchronize(stream));
    }
    n_lmp = np;
    D.lmp_slot = np > 0 ? d_lmp_slot : nullptr;
    D.lmp_mean = d_lmp_mean;
    D.lmp_L = d_lmp_L;
    D.lmp_Lg = d_lmp_Lg;
    return priors_changed();
  }

  // launch with optional programmatic dependent launch (the kernel may start before its predecessor in the stream has
  // finished and orders itself with griddepcontrol.wait) and optional thread-block-cluster dimension
  template <class... KArgs, class... Args>
  int launch_ex(void (*kern)(KArgs...), int grid, int block, size_t smem, bool pdl, int cluster, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (pdl) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
    if (cluster > 1) { at[na].id = cudaLaunchAttributeClusterDimension; at[na].val.clusterDim.x = cluster; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1; ++na; }
    cfg.attrs = at; cfg.numAttrs = na;
    CU(cudaLaunchKernelEx(&cfg, kern, KArgs(args)...));
    ++launches;
    return RBA_OK;
  }
  int tile_grid(int max_blocks) const { return std::max(1, std::min(max_blocks, (D.ntiles + TILE_WARPS - 1) / TILE_WARPS)); }
  int grid_for(long long work_items, int per_block, int blocks_per_sm) const {
    long long g = (work_items + per_block - 1) / per_block;
    g = std::min<long long>(g, (long long)sm_count * blocks_per_sm);
    return (int)std::max<long long>(g, 1);
  }

  // deterministic per-camera sum of yobs[slot][9] over a CSR -> dst[9 nc] (+ all-reduce across shards)
  int camera_reduce(const int* slots, const ReduceItem* items, int nitems, const int* item_ptr, S* dst,
                    const S* addend = nullptr, bool reduce_ranks = true) {
    k_cam_reduce<S><<<grid_for(nitems, 8, 8), 256, 0, stream>>>(D.yobs, slots, items, nitems, D.partial, nullptr, 0);
    k_cam_final9<S><<<(9 * nc + 255) / 256, 256, 0, stream>>>(D.partial, item_ptr, nc, dst, addend);
    launches += 2;
    return reduce_ranks ? allreduce(dst, (size_t)9 * nc) : RBA_OK;
  }

  // ------------------------------------------------------------------------------------------
  // ref: solver/linearizor_base.cpp:59-67
  // Every entry point is split into an enqueue half (kernels + asynchronous copies into its OWN pinned slot) and a finish
  // half (after a stream synchronisation): the public calls are enqueue + synchronise + finish, rba_lm_step strings the
  // enqueue halves of a whole LM inner iteration together and synchronises once.
  int compute_error_enqueue() {
    error_enqueued = false;
    if (error_cache_valid && error_cache_version == state_version) return RBA_OK;  // answered from the cache in finish
    int rc = start(ev_error); if (rc) return rc;
    CU(cudaMemsetAsync(d_flags, 0, 4 * sizeof(int), stream));
    k_error<S><<<EBLOCKS, 256, 0, stream>>>(D, ko, d_epart, d_flags);
    k_sum_partials<6><<<1, 256, 0, stream>>>(d_epart, EBLOCKS, d_red);
    launches += 2;
    if (n_lmp > 0) {  // + this shard's landmark priors' 1/2 |L e|^2, BEFORE the sum over the shards (landmark-owned)
      k_prior_cost<<<1, 256, 0, stream>>>(LandmarkPrior<S>{D.lms, d_lmp_lm, d_lmp_mean, d_lmp_L}, n_lmp, d_red, d_flags);
      ++launches;
    }
    rc = allreduce_scalars(6); if (rc) return rc;
    if (has_abs_prior) {  // + sum of 1/2 |L e|^2, once, after the sum over the shards
      k_prior_cost<<<1, 256, 0, stream>>>(camera_prior(), nc, d_red, d_flags);
      ++launches;
    }
    if (n_pairs > 0) {  // + the pair priors' 1/2 |L e|^2, likewise
      k_prior_cost<<<1, 256, 0, stream>>>(pair_prior(), n_pairs, d_red, d_flags);
      ++launches;
    }
    CU(cudaMemcpyAsync(h_res->error, d_red, sizeof(h_res->error), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(h_res->error_flags, d_flags, sizeof(h_res->error_flags), cudaMemcpyDeviceToHost, stream));
    rc = stop(ev_error); if (rc) return rc;
    error_enqueued = true;
    error_enqueue_version = state_version;
    return RBA_OK;
  }
  int compute_error_finish(rba_residual_info* out) {
    // The LM loop evaluates the cost at the end of an accepted step and again, unchanged state, before the next
    // linearisation (the reference's own TODO, bal_bundle_adjustment.cpp:298-301): the evaluation is deterministic, so
    // the second call returns the cached ResidualInfo without touching the GPU.
    if (!error_enqueued) {
      *out = error_cache;
      tm.residual_evaluation_time = 0.0;
      return RBA_OK;
    }
    const double* e = h_res->error;
    out->all_num_obs = (int64_t)llround(e[0]); out->all_error = e[1]; out->all_residual_sum = e[2];
    out->valid_num_obs = (int64_t)llround(e[3]); out->valid_error = e[4]; out->valid_residual_sum = e[5];
    if (h_res->error_flags[1]) { g_err = "a peer rank did not take part in a cross-shard reduction in time (peer-memory exchange timed out)"; return RBA_ERR_NCCL; }
    out->is_numerically_valid = h_res->error_flags[0] ? 0 : 1;
    out->pad_ = 0;
    tm.residual_evaluation_time = elapsed(ev_error);
    error_cache = *out; error_cache_version = error_enqueue_version; error_cache_valid = true;
    return RBA_OK;
  }
  int compute_error(rba_residual_info* out) override {
    int rc = compute_error_enqueue(); if (rc) return rc;
    if (error_enqueued) CU(cudaStreamSynchronize(stream));
    return compute_error_finish(out);
  }

  // ref: solver/linearizor_qr.cpp:78-138 (staged: LinearizationQR::get_stage1, linearization_qr.hpp:634-712)
  int linearize_enqueue() {
    lin_l0 = launches;
    int rc = start(ev_stage1); if (rc) return rc;
    CU(cudaMemsetAsync(d_flags, 0, 4 * sizeof(int), stream));
    // pass A: squared column norms of the weighted pose Jacobians -> pose_jacobian_scaling_
    k_jp_norms<S><<<grid_for(L.nslots, 256, 8), 256, 0, stream>>>(D, ko, d_flags);
    ++launches;
    rc = camera_reduce(d_csr_obs_slots, d_csr_obs_items, n_obs_items, d_csr_obs_item_ptr, D.diag2); if (rc) return rc;
    if (has_abs_prior) {  // prior Jacobian and its column norms (scaling from the whole Jacobian), after the sum over the shards
      k_prior_linearize<S><<<(nc + 127) / 128, 128, 0, stream>>>(D.cams, d_prior_mean, d_prior_L, nc, D.diag2, d_prior_A, d_prior_r);
      ++launches;
    }
    if (n_pairs > 0) {  // pair-prior blocks and their column norms, likewise
      k_pair_linearize<S><<<(n_pairs + 127) / 128, 128, 0, stream>>>(D.cams, d_pair_ij, d_pair_mean, d_pair_L, n_pairs, d_pair_A, d_pair_r);
      k_pair_diag2<S><<<(nc + 127) / 128, 128, 0, stream>>>(d_pair_A, d_pair_ptr, d_pair_item, nc, D.diag2);
      launches += 2;
    }
    k_scaling<S><<<(9 * nc + 255) / 256, 256, 0, stream>>>(D.diag2, D.scaling, 9 * nc, (S)ko.jacobi_eps);
    // pass B: linearize (scaled) + Jl scaling + Householder QR + panel write
    // (+ the landmark priors' column norms, L~ and g: the LMP instances)
    const bool lmp = D.lmp_slot != nullptr;
    auto k1 = opt.use_householder_marginalization ? (lmp ? k_linearize_qr<S, false, true> : k_linearize_qr<S, false>)
                                                  : (lmp ? k_linearize_qr<S, true, true> : k_linearize_qr<S, true>);  // ref: ipp:149-163 selects perform_qr_givens
    k1<<<tile_grid(k1_max_blocks), TILE_WARPS * 32, k1_smem, stream>>>(D, ko, k1_sc, d_flags, order_k1);
    launches += 2;
    if (opt.preconditioner_type == 0 || opt.solver_type == 2) {
      // JACOBI: D (sum Jp^T Jp) D from the stored scaled Jacobians (Power-SC: these blocks are Hpp, sc/linearization_power_sc.hpp:92-128) (ref: ipp:554-569, block_sparse_matrix.hpp:89-100)
      rc = precond_blocks(0, D.jblocks, nullptr, true); if (rc) return rc;
    }
    const bool jac = opt.preconditioner_type == 0 || opt.solver_type == 2;
    if (has_abs_prior) {  // scaled prior Jacobian, A^T A (+ into the JACOBI blocks), A^T r
      k_prior_scale<S><<<(nc + 127) / 128, 128, 0, stream>>>(d_prior_A, d_prior_r, D.scaling, nc, d_prior_H, d_prior_g, jac ? D.jblocks : nullptr);
      ++launches;
    }
    if (n_pairs > 0) {  // scaled pair blocks; their diagonal blocks and A^T r added to the absolute priors', the O_ij of every edge
      k_pair_scale<S><<<(n_pairs + 127) / 128, 128, 0, stream>>>(d_pair_A, d_pair_ij, D.scaling, n_pairs);
      k_pair_accum<S><<<(nc + 127) / 128, 128, 0, stream>>>(d_pair_A, d_pair_r, d_pair_ptr, d_pair_item, nc, (int)has_abs_prior,
                                                            d_prior_H, d_prior_g, jac ? D.jblocks : nullptr, d_pair_O);
      launches += 2;
    }
    if (panel_form) {
      // rows 3..2n-1 of the Q2 panels do not change with lambda: their part of the gradient (ipp:443-466) and of the
      // SCHUR_JACOBI blocks (ipp:520-552) is accumulated once per linearisation (this shard only; the sum over the
      // shards happens in solve() together with the damping-row part)
      const int want_blocks = opt.preconditioner_type == 1 ? 1 : 0;
      k_panel_grad_blocks<S><<<tile_grid(sm_count * 8), TILE_WARPS * 32, 0, stream>>>(D, want_blocks, order_kp);
      ++launches;
      rc = camera_reduce(d_csr_obs_slots, d_csr_obs_items, n_obs_items, d_csr_obs_item_ptr, D.b0, nullptr, false); if (rc) return rc;
      if (want_blocks) { rc = precond_blocks(3, D.blocks0, nullptr, false); if (rc) return rc; }
    }
    rc = allreduce_scalars(0); if (rc) return rc;
    CU(cudaMemcpyAsync(h_res->linearize_flags, d_flags, sizeof(h_res->linearize_flags), cudaMemcpyDeviceToHost, stream));
    rc = stop(ev_stage1); if (rc) return rc;
    linearized = true;  // provisional: linearize_finish withdraws it on a numerical failure
    new_linearization_point = true;
    su_valid = s_valid = false;
    damping_valid = false;
    have_inc = false;
    return RBA_OK;
  }
  int linearize_finish() {
    CU(cudaGetLastError());
    tm.stage1_time = elapsed(ev_stage1);
    tm.kernel_launches = launches - lin_l0;
    if (h_res->linearize_flags[1]) { linearized = false; g_err = "a peer rank did not take part in a cross-shard reduction in time (peer-memory exchange timed out)"; return RBA_ERR_NCCL; }
    if (h_res->linearize_flags[0]) { linearized = false; return RBA_NUMERICAL_FAILURE; }  // reference: CHECK abort (linearizor_qr.cpp:121-122)
    return RBA_OK;
  }
  int linearize() override {
    int rc = linearize_enqueue(); if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    return linearize_finish();
  }

  // per-camera 9x9 blocks: deterministic two-phase sum over the camera-major observation CSR (modes: see k_precond_partial)
  int precond_blocks(int mode, S* dst, const S* addend, bool reduce_ranks) {
    const int g = (n_pb_items + 127) / 128;
    switch (mode) {
      case 0: k_precond_partial<S, 0><<<g, 128, 0, stream>>>(D.jp, (const S*)nullptr, d_csr_obs_slots, d_pb_items, n_pb_items, D.pblk); break;
      case 1: k_precond_partial<S, 1><<<g, 128, 0, stream>>>(D.jp, D.q1d, d_csr_obs_slots, d_pb_items, n_pb_items, D.pblk); break;
      case 2: k_precond_partial<S, 2><<<g, 128, 0, stream>>>(D.dmp, (const S*)nullptr, d_csr_obs_slots, d_pb_items, n_pb_items, D.pblk); break;
      default: k_precond_partial<S, 3><<<g, 128, 0, stream>>>(D.blk0, (const S*)nullptr, d_csr_obs_slots, d_pb_items, n_pb_items, D.pblk); break;
    }
    k_precond_final<S><<<(45 * nc + 255) / 256, 256, 0, stream>>>(D.pblk, d_pb_item_ptr, nc, addend, dst);
    launches += 2;
    return reduce_ranks ? allreduce(dst, (size_t)81 * nc) : RBA_OK;
  }

  // one complete operator application outside PCG: y = sum over the landmarks of P^T P x_red (this shard), per camera in D.y
  int matvec_launch(const S* xvec) {
    matvec_kernels(xvec, nullptr, false);
    return s_valid ? RBA_OK : cam_reduce_final(false, 0, false);
  }
  // operator part of one matvec: yobs = P^T P x_red for every landmark (e0_only: the implicit operator's E_0 x alone);
  // assembled operator: D.y = S x_red, complete
  void matvec_kernels(const S* xvec, const int* done, bool pdl, int e0_only = 0) {
    if (s_valid) {
      launch_ex(k_rcs_spmv<S>, nc, SPMV_WARPS * 32, 0, pdl, 1, (const int*)d_asm_row_ptr, (const int*)d_asm_col, (const S*)d_asm_S, xvec,
                D.y, done, (int)pdl);
      ++tm.matvec_launches;
      return;
    }
    if (implicit_op) {
      const int ntl = (int)L.tiles.size();
      const bool p = pdl && imp_tile_split == ntl;  // a single kernel between the PCG vector step and the reduction
      if (imp_tile_split > 0)
        launch_ex((k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), imp_grid, IMP_WARPS * 32, imp_smem, p, 1, D, imp_tile_split, xvec, done, (int)p, e0_only);
      if (imp_tile_split < ntl)
        launch_ex(k_matvec_implicit<S>, (ntl - imp_tile_split + TILE_WARPS - 1) / TILE_WARPS, TILE_WARPS * 32, 0, false, 1, D, imp_tile_split, xvec, done, 0, e0_only);
      ++tm.matvec_launches;
      return;
    }
    if (L.n_items_large > 0) {
      k_matvec_large<S, K4_WARPS, KPMAX><<<grid_for(L.n_items_large, K4_WARPS, 4), K4_WARPS * 32, k4_smem_small, stream>>>(
          D, d_items, 0, L.n_items_large, L.k4_scratch_per_warp, xvec, done);
      ++launches;
    }
    if (n_dealt > L.n_items_large) {
      const bool p = pdl && L.n_items_large == 0;
      launch_ex(k_matvec_small_tma<S, K4_WARPS, K4_NS, K4_STAGE>, tma_grid, K4_WARPS * 32, K4_SMEM_TMA, p, 1, D, (const MatvecItem*)d_items,
                L.n_items_large, n_dealt, L.k4_scratch_per_warp, xvec, done, (int)p);
    }
    ++tm.matvec_launches;
  }
  // per-camera sums of the operator output into D.y (peers: into every rank's staging area of the peer exchange).  Inside a
  // solve it is launched dependent on its predecessor and returns at once when the solve has ended.
  int cam_reduce_final(bool peers, int seq, bool in_solve) {
    auto kern = peers ? k_cam_reduce_final<S, true> : k_cam_reduce_final<S, false>;
    return launch_ex(kern, grid_for(n_op_items, 8, 8), 256, 0, in_solve, 1, (const S*)D.yobs, op_slots, op_items, n_op_items, op_item_ptr,
                     D.partial, d_cam_cnt, D.y, in_solve ? (const int*)&d_state->done : nullptr, (int)in_solve, pc, seq, nc);
  }
  int pcg_vec(int i, int mode, bool pdl, int is_last, S lambda, bool fused_ar = false, bool from_partials = false) {
    PeerComm c = pc;
    if (!fused_ar) c.nranks = 1;
    if (D.pair_ov) {  // pair priors: O v of the step's vector (v = x in the refresh's second half, else p) into D.pair_ov first
      if (mode != 3) TRY(pair_ov(mode == 2 ? D.x : D.p, pdl));
      return launch_ex(k_pcg_vec<S, true, true>, pcg_cluster, VEC_THREADS, 0, pdl, pcg_cluster, D, d_state, lambda, i, mode, (double)opt.eta,
                       (int)opt.min_linear_solver_iterations, is_last, (int)pdl, c, ar_seq, from_partials ? op_item_ptr : (const int*)nullptr, d_prog);
    }
    auto kern = D.prior_H ? k_pcg_vec<S, true> : k_pcg_vec<S, false>;
    return launch_ex(kern, pcg_cluster, VEC_THREADS, 0, pdl, pcg_cluster, D, d_state, lambda, i, mode, (double)opt.eta,
                     (int)opt.min_linear_solver_iterations, is_last, (int)pdl, c, ar_seq, from_partials ? op_item_ptr : (const int*)nullptr, d_prog);
  }
  // D.pair_ov = sum_j O_ij v_j (k_pair_ov), ahead of the vector step that consumes it
  int pair_ov(const S* v, bool pdl) {
    return launch_ex(k_pair_ov<S>, (9 * nc + 255) / 256, 256, 0, pdl, 1, D, (const PcgState*)d_state, v);
  }
  // The hand-over through per-segment sums is taken when a cluster CTA's share of the cameras fits the vector kernel's
  // register-resident layout (9 ceil(nc / cluster) <= VEC_THREADS VEC_EPT: <= 1808 cameras with a 16-CTA cluster, <= 904
  // with 8); larger camera counts on one GPU (Final-13682) keep the arrival-counter reduction into D.y, the combination that
  // was measured at that size.
  bool pcg_from_partials() const {
    const bool vec_cached = 9 * ((nc + pcg_cluster - 1) / pcg_cluster) <= VEC_THREADS * VEC_EPT;
    return opt.nranks == 1 && pcg_partials && vec_cached;
  }
  // finish one operator application inside PCG (H v for v = p in mode 0/1, x in mode 2) and do the vector step
  int pcg_apply(int i, int mode, int is_last, S lambda) {
    if (s_valid) return pcg_vec(i, mode, true, is_last, lambda);  // k_rcs_spmv has written D.y
    if (pcg_from_partials()) {
      // one GPU: the vector kernel adds the per-segment sums itself (same order as k_cam_reduce_final's last arriver:
      // bit-identical) -- no arrival counters, fences or second pass in the reduction
      TRY(launch_ex(k_cam_reduce<S>, grid_for(n_op_items, 8, 8), 256, 0, true, 1, (const S*)D.yobs, op_slots, op_items, n_op_items, D.partial,
                    (const int*)&d_state->done, 1));
      return pcg_vec(i, mode, true, is_last, lambda, false, true);
    }
    const bool fused = opt.nranks > 1 && peer_ok;
    if (fused) ++ar_seq;
    // NCCL path: k_cam_reduce_final writes y only for cameras that have observations in this shard; D.y is all-reduced IN
    // PLACE, so without this the other cameras would carry the previous iteration's global sum into the next all-reduce
    if (opt.nranks > 1 && !fused) CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));
    TRY(cam_reduce_final(fused, ar_seq, true));
    if (opt.nranks == 1) return pcg_vec(i, mode, true, is_last, lambda);
    if (fused) return pcg_vec(i, mode, true, is_last, lambda, true);
    TRY(allreduce(D.y, (size_t)9 * nc));
    return pcg_vec(i, mode, false, is_last, lambda);
  }
  // Enqueue iterations 1..last in chunks of `chunk` (enqueue(i)); after each chunk the PcgState is copied into one of two
  // pinned slots, and the host waits for the copy of the chunk before and stops once it shows the solve ended.
  template <class F>
  int enqueue_polled(int last, int chunk, F&& enqueue) {
    int i = 1, pending[2] = {0, 0}, slot = 0;
    bool finished = false;
    while (i <= last && !finished) {
      const int chunk_end = std::min(i + chunk - 1, last);
      for (; i <= chunk_end; ++i) TRY(enqueue(i));
      CU(cudaMemcpyAsync(&h_state[slot], d_state, sizeof(PcgState), cudaMemcpyDeviceToHost, stream));
      CU(cudaEventRecord(poll_ev[slot], stream));
      pending[slot] = 1;
      const int other = slot ^ 1;
      if (pending[other]) {
        CU(cudaEventSynchronize(poll_ev[other]));
        pending[other] = 0;
        if (h_state[other].done) finished = true;
      }
      slot = other;
    }
    return RBA_OK;
  }

  // ref: solver/linearizor_qr.cpp:140-265
  // Power-series solve of the reduced camera system (ref: sc/linearization_power_sc.hpp:130-160, driven by
  // solver/linearizor_power_sc.cpp:140-160 with q_tolerance = eta): per term one E_0 application (the implicit operator
  // kernels with e0_only), the per-camera reduction and k_power_vec; the device convergence flag is polled like in PCG.
  int power_enqueue(void* inc_out) {
    TRY(start(ev_pcg));
    CU(cudaMemsetAsync(d_state, 0, sizeof(PcgState), stream));
    const int order = opt.power_order;
    // pair priors: the series on Hpp^-1 (E_0 - O), O p from k_pair_ov ahead of each term (DESIGN.md section 15)
    auto kern = D.pair_ov ? k_power_vec<S, true> : k_power_vec<S, false>;
    TRY(launch_ex(kern, pcg_cluster, VEC_THREADS, 0, false, pcg_cluster, D, d_state, 0, (double)opt.eta, 0, 0));
    TRY(enqueue_polled(order, opt.pcg_check_period, [&](int i) -> int {
      matvec_kernels(D.p, &d_state->done, true, 1);
      TRY(cam_reduce_final(false, 0, true));
      if (D.pair_ov) TRY(pair_ov(D.p, true));
      return launch_ex(kern, pcg_cluster, VEC_THREADS, 0, true, pcg_cluster, D, d_state, i, (double)opt.eta, (int)(i == order), 1);
    }));
    CU(cudaMemcpyAsync(&h_state[0], d_state, sizeof(PcgState), cudaMemcpyDeviceToHost, stream));
    if (inc_out) CU(cudaMemcpyAsync(inc_out, D.inc, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    TRY(stop(ev_pcg));
    have_inc = true;
    new_linearization_point = false;
    return RBA_OK;
  }

  int solve_enqueue(double lambda_d, void* inc_out) {
    if (!linearized) { g_err = "rba_solve called before a successful rba_linearize"; return RBA_ERR_STATE; }
    const S lambda = (S)lambda_d;
    solve_l0 = launches;
    tm.matvec_launches = 0;
    int rc = start(ev_stage2); if (rc) return rc;
    // stage 2: landmark damping + gradient (+ SCHUR_JACOBI blocks)
    // (landmark priors: the LMP instances, DESIGN.md section 17)
    const bool lmp = D.lmp_slot != nullptr;
    if (opt.solver_type != 0) {
      // Schur-complement solvers: landmark eliminated through the normal equations (Cholesky of Jl^T Jl + lambda I)
      auto k = lmp ? k_sc_stage2<S, true> : k_sc_stage2<S>;
      k<<<tile_grid(sm_count * 8), TILE_WARPS * 32, 0, stream>>>(D, lambda);
    } else {
      auto k = panel_form ? (lmp ? k_stage2<S, true, true> : k_stage2<S, true>) : (lmp ? k_stage2<S, false, true> : k_stage2<S, false>);
      k<<<tile_grid(k2_max_blocks), TILE_WARPS * 32, k2_smem, stream>>>(D, lambda, k2_sc, ko.write_panel);
    }
    ++launches;
    s_valid = false;  // S of the previous lambda; rebuilt if this solve runs long enough (solve_enqueue)
    rc = camera_reduce(d_csr_obs_slots, d_csr_obs_items, n_obs_items, d_csr_obs_item_ptr, D.b, panel_form ? D.b0 : nullptr); if (rc) return rc;
    const bool power = opt.solver_type == 2;
    const bool schur = opt.preconditioner_type == 1 && !power;  // Power-SC inverts Hpp = sum Jp^T Jp + lambda I instead
    if (schur) { rc = panel_form ? precond_blocks(2, D.blocks, D.blocks0, true) : precond_blocks(1, D.blocks, nullptr, true); if (rc) return rc; }
    rc = stop(ev_stage2); if (rc) return rc;
    rc = start(ev_precond); if (rc) return rc;
    // pose damping lambda*I added to the blocks, then explicit inverse (ref: linearization_qr.hpp:796-802, linearizor_qr.cpp:228-237)
    // (+ the masking of the held camera parameters, D.cam_fixed; + the camera priors: A^T A into the SCHUR_JACOBI blocks -- the
    // JACOBI blocks hold it already -- and A^T r into b, both after the sum over the shards and before the masking)
    k_precond_invert<S><<<(nc + 63) / 64, 64, 0, stream>>>(schur ? D.blocks : D.jblocks, lambda, nc, schur ? D.blocks : nullptr, D.inv,
                                                           D.cam_fixed, D.b, schur ? (const S*)D.prior_H : nullptr,
                                                           D.prior_H ? (const S*)d_prior_g : nullptr);
    ++launches;
    rc = stop(ev_precond); if (rc) return rc;
    last_lambda = lambda;
    damping_valid = true;
    if (all_cams_fixed) {
      // no free camera parameter: inc = 0 without PCG / power series (whose stopping tests would divide 0 by 0); stage 2
      // above still ran for the damped landmark factors of the back-substitution.  Every rank skips alike.
      rc = start(ev_pcg); if (rc) return rc;
      CU(cudaMemsetAsync(D.inc, 0, (size_t)9 * nc * sizeof(S), stream));
      if (inc_out) CU(cudaMemcpyAsync(inc_out, D.inc, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
      rc = stop(ev_pcg); if (rc) return rc;
      // no copy into h_state is in flight: every entry point synchronises the stream before it returns
      h_state[0] = PcgState{};
      h_state[0].done = 1; h_state[0].term = 1; h_state[0].reason = 2;  // SUCCESS, |b_f| = 0, 0 iterations
      have_inc = true;
      new_linearization_point = false;
      return RBA_OK;
    }
    // k_cam_reduce_final writes D.y only for cameras with observations, and an earlier call may have left other values in
    // the remaining entries (rba_right_multiply stores lambda x there for every camera).  The one-GPU consumers that read
    // D.y (k_power_vec, and k_pcg_vec without the per-segment hand-over) need the operator's 0 for a camera without
    // observations: cleared once per solve, outside the iteration.
    if (opt.nranks == 1 && (power || !pcg_from_partials())) CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));
    if (power) return power_enqueue(inc_out);
    // PCG (ref: cg/conjugate_gradient.hpp:113-298 ; linearizor_base.cpp:81-103)
    rc = start(ev_pcg); if (rc) return rc;
    CU(cudaMemsetAsync(d_state, 0, sizeof(PcgState), stream));
    const int max_it = std::max(opt.max_linear_solver_iterations, 1);
    const int period = opt.residual_reset_period;
    // The vector kernel publishes the number of the last completed iteration and the end of the solve in host-mapped pinned
    // memory (h_prog); the host enqueues at most pcg_check_period iterations beyond that and stops as soon as it sees the
    // end: no copy or event between the kernels of the loop, and at most pcg_check_period no-op iterations after the end
    // (one GPU, and the peer-memory exchange, whose no-op kernels leave before they communicate).
    const int depth = opt.pcg_check_period;
    h_prog[0] = 0; h_prog[1] = 0;  // nothing in flight writes them: the stream has been synchronised since the previous solve
    // The ranks stop enqueueing at slightly different iterations (whenever each sees the end), so the sequence numbers of the
    // operator exchange restart from a per-solve base that every rank computes alike
    ar_seq = (++pcg_solve_id) * (2 * max_it + 4);
    rc = pcg_vec(0, 3, false, 0, lambda); if (rc) return rc;  // x = 0, r = b, z = M^-1 r, rho, p = z
    auto enqueue_iteration = [&](int i) -> int {
      const int is_last = (i == max_it) ? 1 : 0;
      matvec_kernels(D.p, &d_state->done, true);
      if (i % period == 0) {
        int r2 = pcg_apply(i, 1, 0, lambda); if (r2) return r2;
        matvec_kernels(D.x, &d_state->done, true);
        return pcg_apply(i, 2, is_last, lambda);
      }
      return pcg_apply(i, 0, is_last, lambda);
    };
    if (opt.nranks > 1 && !peer_ok) {
      // NCCL exchange: every rank must enqueue the SAME number of all-reduces, so the decision to stop may depend only on
      // the iteration count -- the flag is polled once per chunk of `depth` iterations, one chunk behind
      TRY(enqueue_polled(max_it, depth, enqueue_iteration));
    } else {
      volatile int* prog = h_prog;
      for (int i = 1; i <= max_it; ++i) {
        unsigned spins = 0;
        while (!prog[1] && i - prog[0] > depth) {
          // every 64k polls: has the stream run dry (a launch failed, or the kernels ended without publishing)?  Then do not wait.
          if ((++spins & 0xffffu) == 0 && cudaStreamQuery(stream) != cudaErrorNotReady) break;
        }
        // once the solve has ended (at iteration prog[0], final when prog[1] is seen), exactly `depth` no-op iterations
        // follow it, whatever the host's pace: the enqueued work does not depend on timing
        if (prog[1] && i - prog[0] > depth) break;
        if (asm_on && i == asm_switch) {
          // the solve has run asm_switch - 1 iterations: from here on S x (S_u once per linearisation, then S for lambda)
          if (!su_valid) assemble(0);
          assemble(1);
          su_valid = s_valid = true;
        }
        rc = enqueue_iteration(i); if (rc) return rc;
      }
    }
    CU(cudaMemcpyAsync(&h_state[0], d_state, sizeof(PcgState), cudaMemcpyDeviceToHost, stream));
    if (inc_out) CU(cudaMemcpyAsync(inc_out, D.inc, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    rc = stop(ev_pcg); if (rc) return rc;
    have_inc = true;
    new_linearization_point = false;
    return RBA_OK;
  }
  int solve_finish(rba_cg_summary* cg) {
    CU(cudaGetLastError());
    tm.stage2_time = elapsed(ev_stage2);
    tm.compute_preconditioner_time = elapsed(ev_precond);
    tm.solve_reduced_system_time = elapsed(ev_pcg);
    tm.kernel_launches = launches - solve_l0;
    if (cg) {
      cg->termination_type = h_state[0].term;
      cg->num_iterations = h_state[0].iter;
      cg->reason = h_state[0].reason;
      cg->num_matvecs = h_state[0].iter + h_state[0].iter / opt.residual_reset_period;
    }
    if (h_state[0].reason == 99) {
      g_err = "PCG: a peer rank did not publish its operator output in time (peer-memory exchange timed out)";
      return RBA_ERR_NCCL;
    }
    return RBA_OK;
  }
  int solve(double lambda_d, void* inc_out, rba_cg_summary* cg) override {
    int rc = solve_enqueue(lambda_d, inc_out); if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    return solve_finish(cg);
  }

  // ref: solver/linearizor_qr.cpp:267-291
  int apply_enqueue(const void* inc_host, bool update_cameras) {
    if (!linearized || !damping_valid) { g_err = "rba_apply / rba_back_substitute need rba_linearize + rba_solve first"; return RBA_ERR_STATE; }
    apply_l0 = launches;
    ++state_version;
    if (inc_host) {
      CU(cudaMemcpyAsync(D.inc, inc_host, (size_t)9 * nc * sizeof(S), cudaMemcpyHostToDevice, stream));
      if (D.cam_fixed) {  // the back-substitution must see the increment the cameras receive
        k_mask_fixed_inc<S><<<(9 * nc + 255) / 256, 256, 0, stream>>>(D.inc, D.cam_fixed, nc);
        ++launches;
      }
    } else if (!have_inc) { g_err = "no device-resident increment (none solved since rba_linearize or rba_set_camera_fixed)"; return RBA_ERR_STATE; }
    int rc = start(ev_backsub); if (rc) return rc;
    CU(cudaMemsetAsync(d_flags, 0, 4 * sizeof(int), stream));
    const int grid = std::min(tile_grid(sm_count * 4), EBLOCKS);
    auto kb = D.lmp_slot ? k_back_substitute<S, true> : k_back_substitute<S>;  // + the landmark priors' part of l_diff
    kb<<<grid, TILE_WARPS * 32, 0, stream>>>(D, D.inc, d_epart, d_flags);
    k_sum_partials<1><<<1, 256, 0, stream>>>(d_epart, grid, d_red);
    launches += 2;
    rc = allreduce_scalars(1); if (rc) return rc;
    if (has_abs_prior) {  // the prior part of the model cost change, once, after the sum over the shards
      k_prior_ldiff<<<1, 256, 0, stream>>>(camera_prior(), D.inc, nc, d_red);
      ++launches;
    }
    if (n_pairs > 0) {  // the pair priors' part, likewise
      k_prior_ldiff<<<1, 256, 0, stream>>>(pair_prior(), D.inc, n_pairs, d_red);
      ++launches;
    }
    rc = stop(ev_backsub); if (rc) return rc;
    rc = start(ev_update); if (rc) return rc;
    if (update_cameras) {
      // NOTE: the reference skips the camera update when l_diff is not finite (linearizor_qr.cpp:275-277); the LM loop
      // then rejects the step and restores the backup, so updating unconditionally is equivalent for the caller.
      k_camera_update<S><<<(nc + 127) / 128, 128, 0, stream>>>(D, D.inc);
      ++launches;
    }
    rc = stop(ev_update); if (rc) return rc;
    CU(cudaMemcpyAsync(&h_res->l_diff, d_red, sizeof(double), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(h_res->apply_flags, d_flags, sizeof(h_res->apply_flags), cudaMemcpyDeviceToHost, stream));
    return RBA_OK;
  }
  int apply_finish(void* l_diff_out) {
    CU(cudaGetLastError());
    tm.back_substitution_time = elapsed(ev_backsub);
    tm.update_cameras_time = elapsed(ev_update);
    tm.kernel_launches = launches - apply_l0;
    if (h_res->apply_flags[1]) { g_err = "a peer rank did not take part in a cross-shard reduction in time (peer-memory exchange timed out)"; return RBA_ERR_NCCL; }
    S l = (S)h_res->l_diff;
    int ret = RBA_OK;
    if (h_res->apply_flags[0] || !std::isfinite((double)l)) { l = std::numeric_limits<S>::quiet_NaN(); ret = RBA_NUMERICAL_FAILURE; }
    *(S*)l_diff_out = l;
    return ret;
  }
  int apply(const void* inc_host, void* l_diff_out, bool update_cameras) override {
    int rc = apply_enqueue(inc_host, update_cameras); if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    return apply_finish(l_diff_out);
  }

  // One LM inner iteration with ONE host synchronisation (SURVEY 8f row 2): [linearize] + solve(lambda) + backup + apply with
  // the device-resident increment + compute_error, the enqueue halves back to back.  Same kernels in the same order as the
  // separate calls, hence bit-identical results.  The reference skips apply when the increment is not finite
  // (bal_bundle_adjustment.cpp:360-399); here the step is applied on the device regardless and the caller restores the
  // backup when `solve_failed` is set (the backup is taken inside).
  int lm_step(bool linearize_first, double lambda, rba_lm_step_result* out) override {
    std::memset(out, 0, sizeof(*out));
    int rc;
    if (linearize_first) { rc = linearize_enqueue(); if (rc) return rc; }
    rc = solve_enqueue(lambda, nullptr); if (rc) return rc;
    rc = backup(); if (rc) return rc;
    rc = apply_enqueue(nullptr, true); if (rc) return rc;
    rc = compute_error_enqueue(); if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    if (linearize_first) { rc = linearize_finish(); if (rc) return rc; }  // numerical failure of the linearisation: as rba_linearize
    rc = solve_finish(&out->cg); if (rc) return rc;
    out->solve_failed = out->cg.termination_type == 2 ? 1 : 0;  // FAILURE: the increment is not usable (reference: non-finite inc)
    S l = 0;
    rc = apply_finish(&l);
    if (rc < 0) return rc;
    out->l_diff = (double)l;
    int rc2 = compute_error_finish(&out->cost); if (rc2) return rc2;
    return rc;  // RBA_NUMERICAL_FAILURE when l_diff is not finite (as rba_apply)
  }

  // optimize_lm_ours (solver/bal_bundle_adjustment.cpp:291-521) on top of lm_step; see rba_lm_run in the header
  static double cost_of(const rba_residual_info& r, int optimized_cost) {
    if (optimized_cost == 0) return r.all_error;
    if (optimized_cost == 1) return r.valid_error;
    return r.valid_num_obs > 0 ? r.valid_error / (double)r.valid_num_obs : 0.0;
  }
  int lm_run(const rba_lm_opts* o, int max_steps, rba_lm_iteration* log, int* steps_done, int* terminated_out, rba_stage_timings* totals) override {
    const S min_lambda = (S)(1.0 / o->max_trust_region_radius), max_lambda = (S)(1.0 / o->min_trust_region_radius);
    const S vee_factor = (S)o->vee_factor, initial_vee = (S)o->initial_vee;
    S lam = (S)(1.0 / o->initial_trust_region_radius), vee = initial_vee;
    bool new_outer = true, terminated = false;
    rba_residual_info ri{};
    if (totals) std::memset(totals, 0, sizeof(*totals));
    int it = 0;
    for (; it < max_steps && !terminated; ++it) {
      rba_lm_iteration& L2 = log[it];
      std::memset(&L2, 0, sizeof(L2));
      L2.lambda = (double)lam;
      const bool lin_first = new_outer;
      double dev = 0;
      if (new_outer) {
        int rc = compute_error(&ri); if (rc) return rc;   // answered from the cache after an accepted step
        if (!ri.is_numerically_valid) { g_err = "did not expect numerical failure during linearization"; return RBA_NUMERICAL_FAILURE; }  // :307-308
        dev += tm.residual_evaluation_time;
        if (totals) totals->residual_evaluation_time += tm.residual_evaluation_time;
        new_outer = false;
      }
      rba_lm_step_result r;
      int rc = lm_step(lin_first, (double)lam, &r);
      if (rc < 0) return rc;
      if (lin_first && rc == RBA_NUMERICAL_FAILURE && !linearized) return rc;  // the linearisation itself failed (reference: CHECK abort)
      const double t_step = (lin_first ? tm.stage1_time : 0.0) + tm.stage2_time + tm.compute_preconditioner_time + tm.solve_reduced_system_time +
                            tm.back_substitution_time + tm.update_cameras_time + tm.residual_evaluation_time;
      dev += t_step;
      if (totals) {
        if (lin_first) totals->stage1_time += tm.stage1_time;
        totals->stage2_time += tm.stage2_time; totals->compute_preconditioner_time += tm.compute_preconditioner_time;
        totals->solve_reduced_system_time += tm.solve_reduced_system_time; totals->back_substitution_time += tm.back_substitution_time;
        totals->update_cameras_time += tm.update_cameras_time; totals->residual_evaluation_time += tm.residual_evaluation_time;
        totals->matvec_launches += tm.matvec_launches;
      }
      L2.device_seconds = dev;
      L2.cg_iterations = r.cg.num_iterations; L2.cg_termination = r.cg.termination_type;
      L2.l_diff = r.l_diff;
      L2.cost = std::numeric_limits<double>::quiet_NaN();
      bool success = false;
      if (r.solve_failed) {
        // non-finite increment (:360-399): not applied by the reference; here undone
        rc = restore(); if (rc) return rc;
      } else {
        const S l_diff = (S)r.l_diff;
        const bool ok = std::isfinite((double)l_diff) && r.cost.is_numerically_valid;
        L2.cost = cost_of(r.cost, o->optimized_cost);
        if (ok) {
          const S f_diff = (S)(cost_of(ri, o->optimized_cost) - cost_of(r.cost, o->optimized_cost));
          S ld = l_diff;
          if (o->optimized_cost == 2) ld = (S)(l_diff / (S)ri.valid_num_obs);  // :436-438
          const S q = (S)(f_diff / ld);
          L2.relative_decrease = (double)q;
          success = ld > S(0) && (double)q > o->min_relative_decrease;     // :443-446
          if (success) {
            const double fac = std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * (double)q - 1.0, 3));
            lam = (S)(lam * (S)fac);                                         // :462-466
            lam = std::max(min_lambda, lam);
            vee = initial_vee;
            new_outer = true;
            const double prev = cost_of(ri, o->optimized_cost == 0 ? 0 : 1), cur = cost_of(r.cost, o->optimized_cost == 0 ? 0 : 1);
            terminated = std::fabs(prev - cur) <= o->function_tolerance * cur;  // function_tolerance_reached (:174-201)
          }
        }
        if (!success) { rc = restore(); if (rc) return rc; }
      }
      if (!success) {
        lam = (S)(vee * lam); vee = (S)(vee * vee_factor);                   // :378-379, :499-500
        if (lam > max_lambda) terminated = true;
      }
      L2.accepted = success ? 1 : 0;
      if (it + 1 >= o->max_num_iterations) terminated = true;
      L2.terminated = terminated ? 1 : 0;
    }
    *steps_done = it;
    *terminated_out = terminated ? 1 : 0;
    return RBA_OK;
  }

  int get_timings(rba_stage_timings* out) const override { *out = tm; out->kernel_launches = launches; return RBA_OK; }
  int get_stats(rba_workload_stats* out) const override {
    std::memset(out, 0, sizeof(*out));
    out->num_landmarks_local = L.nl_local;
    out->num_observations_local = L.nobs_local;
    out->sum_n2 = L.sum_n2;
    out->max_n = L.max_n;
    out->num_tiles = (int)L.tiles.size();
    out->panel_scalars = L.panel_scalars;
    out->panel_scalars_algorithmic = 18 * L.sum_n2;
    out->device_bytes = (int64_t)device_bytes;
    // the operator the last solve ended with: the panels, or S (blocks, column indices, row pointers, x read and y written once)
    out->matvec_algorithmic_bytes = s_valid ? (81 * asm_nnzb + 18 * (int64_t)nc) * (int64_t)sizeof(S) + 4 * (asm_nnzb + nc + 1)
                                           : (18 * L.sum_n2 + 18 * L.nobs_local) * (int64_t)sizeof(S) + 4 * L.nobs_local;
    out->landmark_begin = L.lm_begin;
    out->landmark_end = L.lm_end;
    out->num_matvec_items = (int)L.items.size();
    return RBA_OK;
  }

  int get_scaling(void* scaling, void* diag2) override {
    if (scaling) CU(cudaMemcpyAsync(scaling, D.scaling, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    if (diag2) CU(cudaMemcpyAsync(diag2, D.diag2, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  int get_rhs(void* b) override {
    CU(cudaMemcpyAsync(b, D.b, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  int get_precond(void* inv, void* blocks) override {
    if (inv) CU(cudaMemcpyAsync(inv, D.inv, (size_t)81 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    if (blocks) CU(cudaMemcpyAsync(blocks, D.blocks, (size_t)81 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  // ref: qr/linearization_qr.hpp:823-825
  int right_multiply(const void* x, void* y) override {
    if (!linearized || !damping_valid) { g_err = "rba_right_multiply needs rba_linearize + rba_solve first"; return RBA_ERR_STATE; }
    CU(cudaMemcpyAsync(D.z, x, (size_t)9 * nc * sizeof(S), cudaMemcpyHostToDevice, stream));
    CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));  // cameras without observations in this shard are not written
    TRY(matvec_launch(D.z));
    TRY(allreduce(D.y, (size_t)9 * nc));  // no-op on one GPU
    k_pcg_q<S><<<NPART, 128, 0, stream>>>(D, D.y, D.z, D.y, last_lambda);
    ++launches;
    CU(cudaMemcpyAsync(y, D.y, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    CU(cudaGetLastError());
    return RBA_OK;
  }

  int time_matvec(int reps, double* sec) override {
    if (!linearized || !damping_valid) { g_err = "rba_time_matvec needs rba_linearize + rba_solve first"; return RBA_ERR_STATE; }
    TRY(matvec_launch(D.p));  // warm-up
    TRY(start(ev_mv));
    for (int r = 0; r < reps; ++r) TRY(matvec_launch(D.p));
    TRY(stop(ev_mv));
    CU(cudaStreamSynchronize(stream));
    CU(cudaGetLastError());
    *sec = elapsed(ev_mv) / std::max(reps, 1);
    tm.matvec_time = *sec;
    return RBA_OK;
  }

  int timer_start() override { return start(ev_user); }
  int timer_stop(double* sec) override {
    int rc = stop(ev_user); if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    *sec = elapsed(ev_user);
    return RBA_OK;
  }
  void* stream_ptr() override { return (void*)stream; }
  int synchronize() override { CU(cudaStreamSynchronize(stream)); return RBA_OK; }

  // ------------------------------------------------------------------------------------------
  // The assembled operator (assembled.cuh, DESIGN.md section 4): taken with one GPU and the dense operator when its
  // structure passes the size rules (plan_assembled) and its buffers fit in the free device memory; else the panel
  // product.
  int setup_assembled() {
    if (!asm_hook || opt.nranks != 1 || implicit_op) return RBA_OK;
    PairList P;
    const std::string msg = build_pair_list(L, P);
    if (!msg.empty()) { g_err = msg; return RBA_ERR_UNSUPPORTED; }
    AsmPlan A;
    plan_assembled(L, P, sizeof(S), A);
    if (!A.fits) return RBA_OK;
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if ((size_t)A.device_bytes + ((size_t)256 << 20) > free_b) return RBA_OK;  // keep 256 MB for the rest of the handle and the caller
    TRY(upload(&d_asm_terms, A.terms));
    TRY(upload(&d_asm_wpos, P.wpos));
    TRY(upload(&d_asm_blk_ptr, P.blk_ptr));
    TRY(upload(&d_asm_pos, A.pos));
    TRY(upload(&d_asm_row_ptr, A.row_ptr));
    TRY(upload(&d_asm_col, A.col));
    TRY(dalloc(&d_asm_stage, (size_t)A.nt * 81, false));
    TRY(dalloc(&d_asm_Su, (size_t)A.nblk * 81));
    TRY(dalloc(&d_asm_S, (size_t)A.nnzb * 81));
    asm_nt = A.nt; asm_nblk = (int)A.nblk; asm_nnzb = A.nnzb;
    asm_switch = asm_at > 0 ? asm_at : A.switch_iteration;
    asm_on = true;
    return RBA_OK;
  }
  // S_u (stage 1, damping = 0) or S = S_u + the damping rows' part (stage 2, damping = 1)
  void assemble(int damping) {
    const int grid = (int)std::max<long long>(1, std::min<long long>((asm_nt + 23) / 24, (long long)sm_count * 16));
    k_rcs_terms<S><<<grid, 256, 0, stream>>>(D.panel, d_asm_terms, asm_nt, damping, d_asm_stage);
    k_rcs_combine<S><<<(unsigned)((81LL * asm_nblk + 255) / 256), 256, 0, stream>>>(
        d_asm_blk_ptr, d_asm_wpos, asm_nblk, d_asm_stage, damping ? (const S*)d_asm_Su : nullptr,
        damping ? (const int2*)d_asm_pos : nullptr, damping ? d_asm_S : d_asm_Su);
    launches += 2;
  }

  // ------------------------------------------------------------------------------------------
  // Marginal covariances (DESIGN.md section 16).  Nothing of the handle changes: the scratch is allocated for the call and
  // freed before it returns; the state, the linearisation, the increment, the error cache and the timings are not touched.
  // The term lists built at the first call stay on the handle (not counted in device_bytes).
  template <class T>
  int cov_upload(T** p, const std::vector<T>& v) {
    void* q = nullptr;
    CU(cudaMalloc(&q, std::max<size_t>(v.size(), 1) * sizeof(T)));
    allocs.push_back(q);
    if (!v.empty()) CU(cudaMemcpy(q, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    *p = (T*)q;
    return RBA_OK;
  }
  // The term lists of rba_compute_covariance (build_pair_list), built at the first call.
  int cov_build_lists() {
    if (cov_ready) return RBA_OK;
    PairList P;
    const std::string msg = build_pair_list(L, P);
    if (!msg.empty()) { g_err = msg; return RBA_ERR_UNSUPPORTED; }
    TRY(cov_upload(&d_cov_blk_cam, P.blk_cam));
    TRY(cov_upload(&d_cov_blk_ptr, P.blk_ptr));
    TRY(cov_upload(&d_cov_terms, P.terms));
    TRY(cov_upload(&d_cov_lm_slot0, P.slot0));
    TRY(cov_upload(&d_cov_lm_n, P.nn));
    cov_nblk = (int)P.blk_cam.size();
    cov_ready = true;
    return RBA_OK;
  }
  template <bool TA, bool TB>
  void cov_gemm(long long M, long long N, long long K, double alpha, const double* A, long long lda, const double* B, long long ldb,
                double beta, double* C, long long ldc, int lower, int ktri) {
    k_cov_dgemm<TA, TB><<<dim3((unsigned)(M / COV_TB), (unsigned)(N / COV_TB)), 256, 0, stream>>>((int)M, (int)N, (int)K, alpha, A, lda, B,
                                                                                                   ldb, beta, C, ldc, lower, ktri);
  }
  // dst (rows x cols, column-major, ld dld) <- src (ld sld), on the stream
  int cov_copy(double* dst, long long dld, const double* src, long long sld, long long rows, long long cols) {
    CU(cudaMemcpy2DAsync(dst, dld * sizeof(double), src, sld * sizeof(double), rows * sizeof(double), cols, cudaMemcpyDeviceToDevice, stream));
    return RBA_OK;
  }
  int compute_covariance(double* cam_cov, double* lm_cov) override {
    if (!cam_cov && !lm_cov) { g_err = "rba_compute_covariance: cam_cov and lm_cov are both NULL"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.nranks > 1) {
      g_err = "rba_compute_covariance: sharded handles (nranks > 1) are not supported: the reduced camera matrix would need a cross-rank sum";
      return RBA_ERR_UNSUPPORTED;
    }
    TRY(cov_build_lists());
    constexpr long long TB = COV_TB;
    const long long n = 9LL * nc, np = (n + TB - 1) / TB * TB, ns = L.nslots;
    const int nl = L.nl_local, nt = (int)(np / TB);
    size_t total = 0;
    auto carve = [&](size_t bytes) { const size_t o = total; total += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_A = carve((size_t)(np * np) * 8), o_W = carve((size_t)(np * TB) * 8), o_Y = carve((size_t)(np * TB) * 8),
                 o_T = carve((size_t)(TB * TB) * 8), o_d = carve((size_t)np * 8), o_jp = carve((size_t)ns * 18 * 8),
                 o_kb = carve((size_t)ns * 27 * 8), o_wl = carve((size_t)nl * 9 * 8), o_rk = carve((size_t)nl * 4), o_fail = carve(4),
                 o_cam = carve((size_t)nc * 81 * 8), o_lm = carve(lm_cov ? (size_t)nl * 9 * 8 : 0);
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (total > free_b) {
      g_err = "rba_compute_covariance needs " + std::to_string(total) + " bytes of device memory (a dense " + std::to_string(n) + " x " +
              std::to_string(n) + " float64 reduced camera matrix plus scratch); " + std::to_string(free_b) + " bytes are free";
      return RBA_ERR_UNSUPPORTED;
    }
    char* base = nullptr;
    CU(cudaMalloc(&base, total));
    struct CovScratch { char* p; ~CovScratch() { cudaFree(p); } } scratch{base};  // cudaFree waits for the kernels
    double* A = (double*)(base + o_A); double* W = (double*)(base + o_W); double* Y = (double*)(base + o_Y);
    double* Tt = (double*)(base + o_T); double* d = (double*)(base + o_d); double* jp = (double*)(base + o_jp);
    double* kb = (double*)(base + o_kb); double* wl = (double*)(base + o_wl); int* rk = (int*)(base + o_rk);
    int* fail = (int*)(base + o_fail); double* cam_out = (double*)(base + o_cam); double* lm_out = (double*)(base + o_lm);
    // 1.-2. elimination, assembly, priors, held parameters, equilibration
    CU(cudaMemsetAsync(A, 0, (size_t)(np * np) * 8, stream));
    CU(cudaMemsetAsync(fail, 0x7f, 4, stream));
    const int wgrid = std::max(1, std::min((nl + 3) / 4, sm_count * 16));
    if (n_lmp > 0)  // + L^T L of the landmark priors in Hll
      k_cov_landmark<S, true><<<wgrid, 128, 0, stream>>>(D, ko, d_cov_lm_slot0, d_cov_lm_n, nl, jp, kb, wl, rk, d_lmp_of_lm);
    else
      k_cov_landmark<S><<<wgrid, 128, 0, stream>>>(D, ko, d_cov_lm_slot0, d_cov_lm_n, nl, jp, kb, wl, rk);
    k_cov_assemble<<<std::max(1, std::min((cov_nblk + 7) / 8, sm_count * 8)), 256, 0, stream>>>(
        (const int2*)d_cov_blk_cam, d_cov_blk_ptr, (const int2*)d_cov_terms, cov_nblk, jp, kb, A, np);
    if (has_abs_prior || n_pairs > 0)
      k_cov_priors<S><<<(nc + 127) / 128, 128, 0, stream>>>(D.cams, nc, has_abs_prior ? d_prior_mean : nullptr, d_prior_L, d_pair_ij,
                                                            d_pair_mean, d_pair_L, n_pairs > 0 ? d_pair_ptr : nullptr, d_pair_item,
                                                            d_pair_nbr, A, np);
    k_cov_diag<<<(unsigned)((np + 255) / 256), 256, 0, stream>>>(A, np, n, np, D.cam_fixed, d);
    k_cov_equil<<<dim3((unsigned)(np / 32), (unsigned)(np / 8)), dim3(32, 8), 0, stream>>>(A, np, n, np, D.cam_fixed, d);
    // 3a. potrf, right-looking: factor the diagonal tile, panel <- panel L_kk^-T, trailing lower tiles -= panel panel^T
    for (int k = 0; k < nt; ++k) {
      const long long k0 = k * TB, m = np - k0 - TB;
      k_cov_tile_potrf<<<1, 256, 0, stream>>>(A, np, k0, COV_PIVOT_TAU, fail);
      if (m == 0) break;
      k_cov_tile_trtri<<<1, COV_TB, 0, stream>>>(A, np, k0, Tt, TB);
      double* P = A + (k0 + TB) + k0 * np;
      TRY(cov_copy(W, m, P, np, m, TB));
      cov_gemm<false, true>(m, TB, TB, 1.0, W, m, Tt, TB, 0.0, P, np, 0, 0);
      cov_gemm<false, true>(m, m, TB, -1.0, P, np, P, np, 1.0, P + TB * np, np, 1, 0);
    }
    int h_fail = 0;
    CU(cudaMemcpyAsync(&h_fail, fail, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    CU(cudaGetLastError());
    if (h_fail < n) {
      static const char* names[9] = {"tx", "ty", "tz", "rx", "ry", "rz", "f", "k1", "k2"};
      g_err = "rba_compute_covariance: the reduced camera matrix is singular: Cholesky pivot <= " + std::to_string(COV_PIVOT_TAU) +
              " of the equilibrated matrix at camera " + std::to_string(h_fail / 9) + ", increment entry " + std::to_string(h_fail % 9) +
              " (" + names[h_fail % 9] + "). The gauge is not fixed, or a free camera has no observation and no prior: hold parameters "
              "with rba_set_camera_fixed or add priors with rba_set_camera_prior";
      return RBA_NUMERICAL_FAILURE;
    }
    // 3b. trtri, from the last tile: column panel <- -L22^-1 L21 L11^-1 with the already inverted trailing part
    for (int j = nt - 1; j >= 0; --j) {
      const long long j0 = j * TB, m = np - j0 - TB;
      k_cov_tile_trtri<<<1, COV_TB, 0, stream>>>(A, np, j0, Tt, TB);
      if (m > 0) {
        double* P = A + (j0 + TB) + j0 * np;
        TRY(cov_copy(W, m, P, np, m, TB));
        cov_gemm<false, false>(m, TB, m, 1.0, P + TB * np, np, W, m, 0.0, Y, m, 0, 1);
        cov_gemm<false, false>(m, TB, TB, -1.0, Y, m, Tt, TB, 0.0, P, np, 0, 0);
      }
      TRY(cov_copy(A + j0 + j0 * np, np, Tt, TB, TB, TB));
    }
    // 3c. lauum, by row tiles: row <- L_ii^T row, L_ii <- L_ii^T L_ii, row += (rows below)^T (rows below)
    for (int i = 0; i < nt; ++i) {
      const long long r0 = i * TB, kk = np - r0 - TB;
      if (r0 > 0) {
        TRY(cov_copy(W, TB, A + r0, np, TB, r0));
        cov_gemm<true, false>(TB, r0, TB, 1.0, A + r0 + r0 * np, np, W, TB, 0.0, A + r0, np, 0, 0);
      }
      k_cov_tile_lauu2<<<1, 256, 0, stream>>>(A, np, r0);
      if (kk > 0) cov_gemm<true, false>(TB, r0 + TB, kk, 1.0, A + (r0 + TB) + r0 * np, np, A + (r0 + TB), np, 1.0, A + r0, np, 0, 0);
    }
    // 4. extraction
    if (cam_cov) {
      k_cov_cam_out<<<(81 * nc + 255) / 256, 256, 0, stream>>>(A, np, d, D.cam_fixed, nc, cam_out);
      CU(cudaMemcpyAsync(cam_cov, cam_out, (size_t)81 * nc * sizeof(double), cudaMemcpyDeviceToHost, stream));
    }
    if (lm_cov) {
      k_cov_lm_marginal<<<wgrid, 128, 0, stream>>>(A, np, d, D.cam_fixed, D.slot_cam, d_cov_lm_slot0, d_cov_lm_n, nl, kb, wl, rk, lm_out);
      CU(cudaMemcpyAsync(lm_cov, lm_out, (size_t)9 * nl * sizeof(double), cudaMemcpyDeviceToHost, stream));
    }
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }

  // reference-layout view of one landmark block (see header)
  int debug_get_block(int lm, void* out, int rows, int cols, void* jls_out) override {
    if (lm < L.lm_begin || lm >= L.lm_end) { g_err = "landmark not in this shard"; return RBA_ERR_INVALID_ARGUMENT; }
    const int sidx = L.sorted_of_lm[lm - L.lm_begin];
    const TileInfo& T = L.tiles[L.tile_of_sorted[sidx]];
    const int n = T.n, G = T.G, KP = T.KP, g = sidx - T.lm_base;
    const int pad = (4 - (9 * n) % 4) % 4, lm_idx = 9 * n + pad, res_idx = lm_idx + 3;
    if (rows != 2 * n + 3 || cols != res_idx + 1) { g_err = "block dims mismatch"; return RBA_ERR_INVALID_ARGUMENT; }
    if (!D.panel) { g_err = "rba_debug_get_block needs operator_form = 0 (no Q2 panels are stored for the implicit operator)"; return RBA_ERR_UNSUPPORTED; }
    CU(cudaStreamSynchronize(stream));
    std::vector<S> panel((size_t)2 * n * KP * 64), rec((size_t)28 * n), lmk(24);
    const int slot0 = T.slot_base + g * n;
    CU(cudaMemcpy(panel.data(), D.panel + T.panel_off, panel.size() * sizeof(S), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(rec.data(), D.q1d + (size_t)28 * slot0, rec.size() * sizeof(S), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(lmk.data(), D.lmk + (size_t)24 * sidx, 24 * sizeof(S), cudaMemcpyDeviceToHost));
    S* o = (S*)out;
    std::fill(o, o + (size_t)rows * cols, S(0));
    for (int c = 0; c < 9 * n; ++c) {
      const int i = c / 9, p = c % 9;
      for (int m = 0; m < 3; ++m) o[(size_t)m * cols + c] = rec[(size_t)28 * i + 9 * m + p];  // damped Q1^T Jp
      const int pr = c / 2, v = c % 2, k = pr / G, j = pr % G, lane = g * G + j;
      for (int r = 0; r < 2 * n; ++r) o[(size_t)(3 + r) * cols + c] = panel[(((size_t)r * KP + k) * 32 + lane) * 2 + v];
    }
    o[0 * cols + lm_idx] = lmk[9]; o[0 * cols + lm_idx + 1] = lmk[10]; o[0 * cols + lm_idx + 2] = lmk[11];
    o[1 * cols + lm_idx + 1] = lmk[12]; o[1 * cols + lm_idx + 2] = lmk[13]; o[2 * cols + lm_idx + 2] = lmk[14];
    for (int m = 0; m < 3; ++m) o[(size_t)m * cols + res_idx] = lmk[15 + m];
    if (jls_out) for (int d = 0; d < 3; ++d) ((S*)jls_out)[d] = lmk[18 + d];
    return RBA_OK;
  }
};

template <class S>
int create_impl(const rba_problem_view* pv, const rba_solver_opts* o, rba_handle** out) {
  if (!pv || !o || !out) { g_err = "null argument"; return RBA_ERR_INVALID_ARGUMENT; }
  if (pv->num_cameras <= 0 || pv->num_landmarks <= 0 || !pv->lm_obs_offset || !pv->obs_cam_idx || !pv->obs_xy) {
    g_err = "empty problem";
    return RBA_ERR_INVALID_ARGUMENT;
  }
  auto* s = new Solver<S>();
  s->scalar_size = sizeof(S);
  int rc = s->init(pv, o);
  if (rc != RBA_OK) { delete s; return rc; }
  *out = s;
  return RBA_OK;
}

}  // namespace rba

extern "C" {

int32_t rba_abi_version(void) { return RBA_ABI_VERSION; }
const char* rba_last_error(void) { return rba::g_err.c_str(); }

void rba_default_solver_opts(rba_solver_opts* o) {
  std::memset(o, 0, sizeof(*o));
  o->use_householder_marginalization = 1;
  o->use_valid_projections_only = 0;
  o->robust_norm = 0;
  o->huber_parameter = 1.0;
  o->jacobi_scaling_epsilon = 0.0;
  o->preconditioner_type = 1;
  o->min_linear_solver_iterations = 0;
  o->max_linear_solver_iterations = 500;
  o->eta = 0.1;
  o->residual_reset_period = 10;
  o->device = -1;
  o->rank = 0;
  o->nranks = 1;
  o->pcg_check_period = 4;
  o->use_cuda_graphs = 0;
  o->power_order = 20;
}

int32_t rba_create_f32(const rba_problem_view* p, const rba_solver_opts* o, rba_handle** out) { return rba::create_impl<float>(p, o, out); }
int32_t rba_create_f64(const rba_problem_view* p, const rba_solver_opts* o, rba_handle** out) { return rba::create_impl<double>(p, o, out); }
int32_t rba_destroy(rba_handle* h) { delete h; return RBA_OK; }
int32_t rba_get_workload_stats(const rba_handle* h, rba_workload_stats* out) { return h->get_stats(out); }
int32_t rba_scalar_size(const rba_handle* h) { return h->scalar_size; }

int32_t rba_partition_landmarks(int32_t nl, const int64_t* off, int32_t nranks, int32_t* bounds) {
  if (nl <= 0 || nranks <= 0 || !off || !bounds) return RBA_ERR_INVALID_ARGUMENT;
  rba::partition_landmarks(nl, off, nranks, bounds);
  return RBA_OK;
}

// ---- BAL loader (host only) ----
struct rba_bal_file {
  rootba_b200::BalProblemSoA<double> p;
  double timings[5] = {0, 0, 0, 0, 0};
};

int32_t rba_bal_load(const char* path, int32_t normalize, double scale, int32_t num_threads, rba_bal_file** out) {
  if (!path || !out) { rba::g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }
  *out = nullptr;
  try {
    std::unique_ptr<rba_bal_file> f(new rba_bal_file());
    rootba_b200::LoadTimings t;
    if (rootba_b200::detail::is_bundler_file(path)) f->p = rootba_b200::load_bundler_soa(path, num_threads);  // autodetect_input_type
    else f->p = rootba_b200::load_bal_parallel(path, num_threads, &t);
    const auto t0 = std::chrono::steady_clock::now();
    if (normalize) f->p.normalize(scale);
    f->timings[0] = t.read; f->timings[1] = t.count; f->timings[2] = t.parse; f->timings[3] = t.csr;
    f->timings[4] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    *out = f.release();
    return RBA_OK;
  } catch (const std::exception& e) {
    rba::g_err = e.what();
    return RBA_ERR_INVALID_ARGUMENT;
  }
}
int32_t rba_bal_filter_obs(rba_bal_file* f, double threshold) {
  if (!f || threshold < 0) { rba::g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }  // the reference CHECK_GEs the threshold
  f->p.filter_obs(threshold);
  return RBA_OK;
}
int32_t rba_bal_perturb(rba_bal_file* f, double rotation_sigma, double translation_sigma, double point_sigma, int32_t seed) {
  if (!f || rotation_sigma < 0 || translation_sigma < 0 || point_sigma < 0) { rba::g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }  // reference: CHECK_GE
  f->p.perturb(rotation_sigma, translation_sigma, point_sigma, seed);
  return RBA_OK;
}
int32_t rba_bal_dims(const rba_bal_file* f, int32_t* nc, int32_t* nl, int64_t* nobs) {
  if (!f) return RBA_ERR_INVALID_ARGUMENT;
  if (nc) *nc = f->p.nc;
  if (nl) *nl = f->p.nl;
  if (nobs) *nobs = f->p.num_observations();
  return RBA_OK;
}
int32_t rba_bal_copy(const rba_bal_file* f, double* cams, double* lms, int64_t* off, int32_t* oc, double* xy) {
  if (!f) return RBA_ERR_INVALID_ARGUMENT;
  if (cams) std::copy(f->p.cams.begin(), f->p.cams.end(), cams);
  if (lms) std::copy(f->p.lms.begin(), f->p.lms.end(), lms);
  if (off) std::copy(f->p.lm_off.begin(), f->p.lm_off.end(), off);
  if (oc) std::copy(f->p.obs_cam.begin(), f->p.obs_cam.end(), oc);
  if (xy) std::copy(f->p.obs_xy.begin(), f->p.obs_xy.end(), xy);
  return RBA_OK;
}
int32_t rba_bal_load_timings(const rba_bal_file* f, double* out5) {
  if (!f || !out5) return RBA_ERR_INVALID_ARGUMENT;
  std::copy(f->timings, f->timings + 5, out5);
  return RBA_OK;
}
int32_t rba_bal_free(rba_bal_file* f) { delete f; return RBA_OK; }

int32_t rba_layout_selftest(const rba_problem_view* pv, int32_t rank, int32_t nranks, int32_t scalar_size) {
  using namespace rba;
  if (!pv || nranks < 1 || rank < 0 || rank >= nranks) { g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }
  Layout L;
  std::string msg = build_layout(pv->num_cameras, pv->num_landmarks, pv->lm_obs_offset, pv->obs_cam_idx, rank, nranks, scalar_size == 4 ? 16 : 10, L);
  if (!msg.empty()) { g_err = msg; return RBA_ERR_INVALID_ARGUMENT; }
  auto fail = [&](const std::string& m) { g_err = "layout selftest: " + m; return RBA_ERR_STATE; };
  // observations <-> slots
  std::vector<char> seen((size_t)L.nobs_local, 0);
  const int64_t obs0 = pv->lm_obs_offset[L.lm_begin];
  long long real_slots = 0;
  for (int s = 0; s < L.nslots; ++s) {
    if (L.slot_lm[s] < 0) { if (L.slot_obs[s] >= 0) return fail("padding slot with an observation"); continue; }
    const long long o = L.slot_obs[s];
    if (o < obs0 || o - obs0 >= L.nobs_local) return fail("slot observation outside the shard");
    if (seen[o - obs0]++) return fail("observation assigned twice");
    if (pv->obs_cam_idx[o] != L.slot_cam[s]) return fail("slot camera mismatch");
    const int lm = L.lm_begin + L.slot_lm[s];
    if (o < pv->lm_obs_offset[lm] || o >= pv->lm_obs_offset[lm + 1]) return fail("slot landmark mismatch");
    ++real_slots;
  }
  if (real_slots != L.nobs_local) return fail("not every observation has a slot");
  // tiles
  std::vector<char> lm_seen((size_t)L.nl_local, 0);
  long long panel = 0;
  for (size_t t = 0; t < L.tiles.size(); ++t) {
    const TileInfo& T = L.tiles[t];
    const int W = 32 / T.G;
    if (T.G != group_size_for(T.n) || T.KP != kp_for(T.n, T.G) || 2 * T.G * T.KP < 9 * T.n) return fail("tile class");
    if (T.panel_off != panel) return fail("panel offsets are not contiguous");
    panel += (long long)2 * T.n * T.KP * 64;
    for (int g = 0; g < W; ++g) {
      const int lm = L.sorted_lm[T.lm_base + g];
      if ((g < T.nvalid) != (lm >= 0)) return fail("nvalid");
      if (lm < 0) continue;
      if (lm_seen[lm]++) return fail("landmark in two tiles");
      if (pv->lm_obs_offset[L.lm_begin + lm + 1] - pv->lm_obs_offset[L.lm_begin + lm] != T.n) return fail("track length of tile");
      for (int i = 0; i < T.n; ++i) {
        const int s = T.slot_base + g * T.n + i;
        if (L.slot_lm[s] != lm || L.slot_obs[s] != pv->lm_obs_offset[L.lm_begin + lm] + i) return fail("slot order inside a landmark");
      }
      if (L.sorted_of_lm[lm] != T.lm_base + g) return fail("sorted_of_lm");
    }
  }
  if (panel != L.panel_scalars) return fail("panel size");
  for (char c : lm_seen) if (!c) return fail("landmark without tile");
  // matvec items: row chunks tile [0, 2n) of every tile exactly once; y slots
  std::vector<int> rows_covered(L.tiles.size(), 0);
  std::vector<char> yslot_used((size_t)L.nyslots, 0);
  for (const MatvecItem& it : L.items) {
    const TileInfo& T = L.tiles[it.tile];
    if (it.nrows <= 0 || it.row0 < 0 || it.row0 + it.nrows > 2 * T.n) return fail("item rows");
    rows_covered[it.tile] += it.nrows;
    for (int k = 0; k < (32 / T.G) * T.n; ++k) {
      if (it.yslot_base + k >= L.nyslots) return fail("y slot range");
      if (yslot_used[it.yslot_base + k]++) return fail("y slot written by two items");
    }
  }
  for (size_t t = 0; t < L.tiles.size(); ++t) if (rows_covered[t] != 2 * L.tiles[t].n) return fail("rows not covered exactly once");
  // camera CSRs
  auto check_csr = [&](const CameraCSR& C, long long expect) -> bool {
    if ((long long)C.slots.size() != expect) return false;
    for (int c = 0; c < pv->num_cameras; ++c) {
      for (int e = C.cam_ptr[c]; e < C.cam_ptr[c + 1]; ++e) if (e > C.cam_ptr[c] && C.slots[e] <= C.slots[e - 1]) return false;
      int covered = 0;
      for (int q = C.cam_item_ptr[c]; q < C.cam_item_ptr[c + 1]; ++q) {
        if (C.items[q].cam != c || C.items[q].begin != C.cam_ptr[c] + covered) return false;
        covered += C.items[q].end - C.items[q].begin;
      }
      if (covered != C.cam_ptr[c + 1] - C.cam_ptr[c]) return false;
    }
    return true;
  };
  if (!check_csr(L.csr_obs, L.nobs_local)) return fail("observation CSR");
  for (int c = 0; c < pv->num_cameras; ++c)
    for (int e = L.csr_obs.cam_ptr[c]; e < L.csr_obs.cam_ptr[c + 1]; ++e)
      if (L.slot_cam[L.csr_obs.slots[e]] != c || L.slot_lm[L.csr_obs.slots[e]] < 0) return fail("observation CSR camera");
  if (!L.csr_y_is_obs) {
    long long expect = 0;
    for (const MatvecItem& it : L.items) expect += (long long)L.tiles[it.tile].nvalid * L.tiles[it.tile].n;
    if (!check_csr(L.csr_y, expect)) return fail("y CSR");
  }
  return RBA_OK;
}

int32_t rba_set_state(rba_handle* h, const void* cams, const void* lms) { return h->set_state(cams, lms); }
int32_t rba_get_state(rba_handle* h, void* cams, void* lms) { return h->get_state(cams, lms); }
int32_t rba_backup(rba_handle* h) { return h->backup(); }
int32_t rba_restore(rba_handle* h) { return h->restore(); }
int32_t rba_set_camera_fixed(rba_handle* h, const uint8_t* flags) { return h->set_camera_fixed(flags); }
int32_t rba_set_camera_prior(rba_handle* h, const void* mean, const void* sqrt_info) { return h->set_camera_prior(mean, sqrt_info); }
int32_t rba_set_camera_pair_prior(rba_handle* h, int32_t num_pairs, const int32_t* pairs, const void* mean, const void* sqrt_info) {
  return h->set_camera_pair_prior(num_pairs, pairs, mean, sqrt_info);
}
int32_t rba_set_landmark_prior(rba_handle* h, int32_t num, const int32_t* lm_idx, const void* mean, const void* sqrt_info) {
  return h->set_landmark_prior(num, lm_idx, mean, sqrt_info);
}
int32_t rba_compute_error(rba_handle* h, rba_residual_info* out) { return h->compute_error(out); }
int32_t rba_linearize(rba_handle* h) { return h->linearize(); }

#define CHECK_TYPE(h, sz) \
  if ((h)->scalar_size != (sz)) { rba::g_err = "scalar type of the handle does not match the entry point"; return RBA_ERR_INVALID_ARGUMENT; }

int32_t rba_solve_f32(rba_handle* h, float lambda, float* inc, rba_cg_summary* cg) { CHECK_TYPE(h, 4); return h->solve(lambda, inc, cg); }
int32_t rba_solve_f64(rba_handle* h, double lambda, double* inc, rba_cg_summary* cg) { CHECK_TYPE(h, 8); return h->solve(lambda, inc, cg); }
int32_t rba_apply_f32(rba_handle* h, const float* inc, float* l) { CHECK_TYPE(h, 4); return h->apply(inc, l, true); }
int32_t rba_apply_f64(rba_handle* h, const double* inc, double* l) { CHECK_TYPE(h, 8); return h->apply(inc, l, true); }
int32_t rba_lm_step_f32(rba_handle* h, int32_t linearize_first, float lambda, rba_lm_step_result* out) { CHECK_TYPE(h, 4); return h->lm_step(linearize_first != 0, lambda, out); }
int32_t rba_lm_step_f64(rba_handle* h, int32_t linearize_first, double lambda, rba_lm_step_result* out) { CHECK_TYPE(h, 8); return h->lm_step(linearize_first != 0, lambda, out); }
void rba_default_lm_opts(rba_lm_opts* o) {  /* defaults of SolverOptions (solver_options.hpp) */
  o->initial_trust_region_radius = 1e4; o->min_trust_region_radius = 1e-32; o->max_trust_region_radius = 1e16;
  o->min_relative_decrease = 0.0; o->initial_vee = 2.0; o->vee_factor = 2.0; o->function_tolerance = 1e-6;
  o->max_num_iterations = 20; o->optimized_cost = 0;
}
int32_t rba_lm_run_f32(rba_handle* h, const rba_lm_opts* o, int32_t max_steps, rba_lm_iteration* log, int32_t* steps_done, int32_t* terminated, rba_stage_timings* totals) {
  CHECK_TYPE(h, 4); if (!o || !log || !steps_done || !terminated || max_steps < 0) { rba::g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }
  return h->lm_run(o, max_steps, log, steps_done, terminated, totals);
}
int32_t rba_lm_run_f64(rba_handle* h, const rba_lm_opts* o, int32_t max_steps, rba_lm_iteration* log, int32_t* steps_done, int32_t* terminated, rba_stage_timings* totals) {
  CHECK_TYPE(h, 8); if (!o || !log || !steps_done || !terminated || max_steps < 0) { rba::g_err = "bad arguments"; return RBA_ERR_INVALID_ARGUMENT; }
  return h->lm_run(o, max_steps, log, steps_done, terminated, totals);
}
int32_t rba_back_substitute_f32(rba_handle* h, const float* inc, float* l) { CHECK_TYPE(h, 4); return h->apply(inc, l, false); }
int32_t rba_back_substitute_f64(rba_handle* h, const double* inc, double* l) { CHECK_TYPE(h, 8); return h->apply(inc, l, false); }
int32_t rba_get_timings(const rba_handle* h, rba_stage_timings* out) { return h->get_timings(out); }
int32_t rba_get_jacobian_scaling(rba_handle* h, void* s, void* d) { return h->get_scaling(s, d); }
int32_t rba_get_rhs(rba_handle* h, void* b) { return h->get_rhs(b); }
int32_t rba_get_preconditioner(rba_handle* h, void* inv, void* blocks) { return h->get_precond(inv, blocks); }
int32_t rba_right_multiply(rba_handle* h, const void* x, void* y) { return h->right_multiply(x, y); }
int32_t rba_debug_get_block(rba_handle* h, int32_t lm, void* out, int32_t rows, int32_t cols, void* jls) {
  return h->debug_get_block(lm, out, rows, cols, jls);
}
int32_t rba_compute_covariance(rba_handle* h, double* cam_cov, double* lm_cov) { return h->compute_covariance(cam_cov, lm_cov); }
int32_t rba_time_matvec(rba_handle* h, int32_t reps, double* sec) { return h->time_matvec(reps, sec); }
int32_t rba_timer_start(rba_handle* h) { return h->timer_start(); }
int32_t rba_timer_stop(rba_handle* h, double* sec) { return h->timer_stop(sec); }
void* rba_stream(rba_handle* h) { return h->stream_ptr(); }
int32_t rba_synchronize(rba_handle* h) { return h->synchronize(); }

int32_t rba_nccl_unique_id(void* out128) {
  rba::NcclApi* api = rba::nccl_api();
  if (!api) { rba::g_err = "libnccl.so.2 could not be loaded"; return RBA_ERR_NCCL; }
  ncclUniqueId id;
  ncclResult_t r = api->GetUniqueId(&id);
  if (r != ncclSuccess) { rba::g_err = std::string("ncclGetUniqueId: ") + api->GetErrorString(r); return RBA_ERR_NCCL; }
  std::memcpy(out128, &id, sizeof(id));
  return RBA_OK;
}
int32_t rba_comm_init(rba_handle* h, const void* uid) { return h->comm_init(uid); }
int32_t rba_ipc_export(rba_handle* h, void* out128) { return h->ipc_export(out128); }
int32_t rba_ipc_import(rba_handle* h, const void* all) { return h->ipc_import(all); }

}  // extern "C"
