// Host orchestration + C ABI (include/rootba_b200.h) of the H100-native square-root BA inner loop.
// One rba_handle = one landmark shard on one GPU; everything is enqueued on one CUDA stream.
// "ref:" citations are relative to src/rootba/ of the reference (NikolausDemmel/rootba @ d3900037).
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <array>
#include <limits>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rootba_b200.h"
#include "../host/bal_io_fast.hpp"
#include "kernels.cuh"
#include "covariance.cuh"
#include "dense_solve.cuh"
#include "cluster_precond.cuh"
#include "assembled.cuh"
#include "rigs.cuh"
#include "triangulate.cuh"
#include "resect.cuh"
#include "nccl_dyn.hpp"

namespace rba {

thread_local std::string g_err;

// the host builds the pair lists as IntPair (layout.hpp); the kernels read them as int2
static_assert(sizeof(IntPair) == sizeof(int2), "IntPair must have the layout of int2");
static_assert(RBA_CLUSTER_MAX_CAMERAS == CLUSTER_MAX_CAMERAS, "the header and the layout agree on the largest cluster");
static_assert(sizeof(rba_triangulate_opts) == 32, "rba_triangulate_opts is 32 bytes without implicit padding");
static_assert(sizeof(rba_resect_opts) == 24, "rba_resect_opts is 24 bytes without implicit padding");

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

// Owns one cudaMalloc'd array of `size()` entries (Solver::alloc makes them) and frees it with itself.  Move-only.
template <class T>
class DeviceBuffer {
  T* p_ = nullptr; size_t n_ = 0;
 public:
  DeviceBuffer() = default;
  DeviceBuffer(T* p, size_t n) : p_(p), n_(n) {}
  DeviceBuffer(DeviceBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }  // o frees the old array
  ~DeviceBuffer() { if (p_) cudaFree(p_); }
  T* get() const { return p_; }
  size_t size() const { return n_; }  // the entries asked for
  void take(DeviceBuffer& o) { if (o.p_) *this = std::move(o); }  // a setter's commit: o's array, if it has one
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
  virtual int set_intrinsics_groups(const int32_t* group) = 0;
  virtual int set_camera_rigs(const int32_t* rig, const void* cam_from_rig) = 0;
  virtual int set_rig_sensors(const int32_t* sensor) = 0;
  virtual int get_rig_extrinsics(void* cam_from_rig) = 0;
  virtual int set_observation_info(const void* sqrt_info) = 0;
  virtual int set_observation_loss(const uint8_t* kind, const void* scale) = 0;
  virtual int set_prior_loss(int32_t prior_kind, int32_t num, const uint8_t* kind, const void* scale) = 0;
  virtual int get_prior_residuals(int32_t prior_kind, void* residual, void* robust_weight) = 0;
  virtual int get_observation_residuals(void* residual, void* robust_weight, uint8_t* flags) = 0;
  virtual int triangulate(const rba_triangulate_opts* o, int32_t num, const int32_t* lm_idx, uint8_t* status, double* angle,
                          double* cost) = 0;
  virtual int resect(const rba_resect_opts* o, int32_t num, const int32_t* cam_idx, uint8_t* status, int32_t* points,
                     double* cost) = 0;
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
  virtual int set_camera_clusters(const int32_t* cluster_of) = 0;
  virtual int get_cluster_precond(int32_t* cluster_of, double* blocks, int32_t* status) = 0;
  virtual int right_multiply(const void* x, void* y) = 0;
  virtual int debug_get_block(int lm, void* out, int rows, int cols, void* jls) = 0;
  virtual int compute_covariance(double* cam_cov, double* lm_cov) = 0;
  virtual int compute_covariance_blocks(const rba_covariance_query* q) = 0;
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
  long long nobs_total = 0;        // observations of the full problem (every shard)
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::vector<DeviceBuffer<char>> owned;  // the buffers of set-up (dalloc), freed with the handle
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
  // the Q2 panels exist: the dense operator (k_matvec_small_tma, k_matvec_large) stores and reads them; the implicit
  // operator, which the Schur-complement solvers share, has none (validate_options)
  bool panels = true;
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
  // The problem terms of the setters.  A setter fills the term's buffers while the new lists fit in them (their size is the
  // capacity), else new ones in a local term, which it adopts once every buffer exists and is filled: a failed call leaves
  // the previous term in force.  point_at_terms derives the kernels' pointers from the terms.
  struct HeldTerm {                // rba_set_camera_fixed; D.cam_fixed = flags while any flag is set
    std::vector<uint8_t> host;     // [nc] the flags, empty = none
    DeviceBuffer<uint8_t> flags;   // [nc]
    bool all = false;              // no free camera parameter: the reduced system is empty and its solve is skipped
  } held;
  // The robust losses of one prior kind (rba_set_prior_loss, DESIGN.md section 22), owned by its term: on while an item of the
  // term has a loss other than NONE.  The setters of the kind clear them (on = false).
  struct PriorLoss {
    bool on = false;
    DeviceBuffer<S> rec;           // the loss records of the term's n items (loss_records layout, read by slot_loss)
    DeviceBuffer<S> Lw;            // sqrt(w) L of the last linearisation (k_prior_weight), read in place of L
  };
  struct CameraPriorTerm {         // rba_set_camera_prior, DESIGN.md section 14; D.prior_H = H while there are absolute or pair priors
    bool on = false;               // any L_c is non-zero
    PriorLoss loss;                // item = camera
    DeviceBuffer<S> mean;          // [nc][10] mean, quaternion normalised
    DeviceBuffer<S> L;             // [nc][81] square-root information
    DeviceBuffer<S> A;             // [nc][81] L de/d(inc): unscaled after k_prior_linearize, scaled after k_prior_scale
    DeviceBuffer<S> r;             // [nc][9]  L e at the linearisation point
    DeviceBuffer<S> H;             // [nc][81] A^T A (+ the pair priors' diagonal blocks)
    DeviceBuffer<S> g;             // [nc][9]  A^T r (+ the pair priors' A_s^T r)
    void adopt(CameraPriorTerm& o) { mean.take(o.mean); L.take(o.L); A.take(o.A); r.take(o.r); H.take(o.H); g.take(o.g); }
  } cprior;
  struct PairPriorTerm {           // rba_set_camera_pair_prior, DESIGN.md section 15; D.pair_ov set while n > 0
    int n = 0;                     // pairs with a non-zero L (m: the capacity)
    std::vector<int> item_of;      // [num_pairs of the last call] the pair's index among the n, -1 = dropped (all-zero L)
    PriorLoss loss;
    DeviceBuffer<int> ij;          // [m][2] cameras (i, j)
    DeviceBuffer<S> mean;          // [m][7] R0 quaternion (normalised), t0
    DeviceBuffer<S> L;             // [m][36] square-root information
    DeviceBuffer<S> A;             // [m][2][36] pose blocks A_i, A_j: unscaled after k_pair_linearize, scaled after k_pair_scale
    DeviceBuffer<S> r;             // [m][6] L e at the linearisation point
    DeviceBuffer<int> item;        // [2m] incident sides 2 p + side, camera-major (CSR ptr)
    DeviceBuffer<int> nbr;         // [2m] the other camera of each side
    DeviceBuffer<S> O;             // [2m][36] O of each directed edge
    DeviceBuffer<int> ptr;         // [nc + 1]
    DeviceBuffer<S> ov;            // [9 nc]
    void adopt(PairPriorTerm& o) { ij.take(o.ij); mean.take(o.mean); L.take(o.L); A.take(o.A); r.take(o.r); item.take(o.item);
                                   nbr.take(o.nbr); O.take(o.O); ptr.take(o.ptr); ov.take(o.ov); }
  } pprior;
  struct LandmarkPriorTerm {       // rba_set_landmark_prior, DESIGN.md section 17; D.lmp_slot set while n > 0
    int n = 0;                     // priors of this shard with a non-zero L (m: the capacity)
    std::vector<int> item_of;      // [num of the last call] the prior's index among the n, -1 = dropped (all-zero L), -2 = other shard
    PriorLoss loss;
    DeviceBuffer<int> slot;        // [nsorted] prior slot per sorted landmark, -1 = none
    DeviceBuffer<int> of_lm;       // [nl_local] prior slot per local landmark, -1 = none (rba_compute_covariance)
    DeviceBuffer<int> lm;          // [m] local landmark of each prior
    DeviceBuffer<S> mean, L, Lg;   // [m][3], [m][9], [m][12]
    void adopt(LandmarkPriorTerm& o) { slot.take(o.slot); of_lm.take(o.of_lm); lm.take(o.lm); mean.take(o.mean); L.take(o.L); Lg.take(o.Lg); }
  } lprior;
  struct GroupTerm {               // rba_set_intrinsics_groups, DESIGN.md section 18
    int n = 0;                     // groups of >= 2 cameras; 0 = the unmodified path
    std::vector<int> host_lead;    // [nc] lead of the camera's group, -1 = own intrinsics (also a group of one)
    DeviceBuffer<int> lead, ptr, mem;  // new lists ({} to fit) at every call with groups
    DeviceBuffer<uint8_t> fixed;   // [nc] the user's flags + RBA_FIX_INTRINSICS on every member but the lead
    DeviceBuffer<S> ve, y;         // [9 nc] the expanded operator input P v, the contracted output the vector step reads
    void adopt(GroupTerm& o) { lead.take(o.lead); ptr.take(o.ptr); mem.take(o.mem); fixed.take(o.fixed); ve.take(o.ve); y.take(o.y); }
  } grp;
  struct RigTerm {                 // rba_set_camera_rigs, DESIGN.md section 23
    int n = 0;                     // rigs of >= 2 cameras; 0 = the unmodified path
    std::vector<int> host_lead;    // [nc] lead of the camera's rig, -1 = free camera (also a rig of one)
    std::vector<int> host_first;   // [nc] the rig's lowest-index camera (its lead without sensors), -1 likewise
    std::vector<double> host_E;    // [nc][7] the extrinsics given, quaternion normalised
    DeviceBuffer<int> lead, ptr, mem;  // new lists ({} to fit) at every call with rigs
    DeviceBuffer<S> adj;           // [nc][36] A_j
    DeviceBuffer<double> M;        // [nc][7] M_j = E_j E_lead^-1
    DeviceBuffer<S> pt;            // [nc][36] P~_j of the last linearisation
    DeviceBuffer<S> du;            // [nr][6] D_u of the last linearisation
    DeviceBuffer<uint8_t> fixed;   // [nc] the user's flags + RBA_FIX_POSE on every member but the lead (+ the groups' bits)
    DeviceBuffer<S> ve, y;         // [9 nc] the expanded operator input P~ v, the contracted output the vector step reads
    void adopt(RigTerm& o) { lead.take(o.lead); ptr.take(o.ptr); mem.take(o.mem); adj.take(o.adj); M.take(o.M); pt.take(o.pt);
                             du.take(o.du); fixed.take(o.fixed); ve.take(o.ve); y.take(o.y); }
  } rig;
  struct SensorTerm {              // rba_set_rig_sensors, DESIGN.md section 24
    int n = 0;                     // sensors; 0 = rigs as in section 23
    std::vector<int> host_home;    // [nc] the home of the camera's sensor, -1 = held extrinsics
    DeviceBuffer<int> home, ptr, mem;  // new lists ({} to fit) at every call with sensors
    DeviceBuffer<double> K;        // [nc][7] E_lead(home) E_lead(j)^-1
    DeviceBuffer<S> qt, ds;        // [nc][6] Q~_j, [ns][6] D_s of the last linearisation
    DeviceBuffer<uint8_t> cam_fixed;  // [nc] the user's flags without RBA_FIX_POSE on sensor cameras (D.cam_fixed)
    DeviceBuffer<S> blk, b;        // [81 nc], [9 nc] the inputs of k_rig_precond, which writes D.blocks and D.b
    void adopt(SensorTerm& o) { home.take(o.home); ptr.take(o.ptr); mem.take(o.mem); K.take(o.K); qt.take(o.qt); ds.take(o.ds);
                                cam_fixed.take(o.cam_fixed); blk.take(o.blk); b.take(o.b); }
  } sen;
  struct ObservationTerm {
    bool on = false;               // rba_set_observation_info, DESIGN.md section 19: W [nslots][4] = D.obs_W while on
    DeviceBuffer<S> W;
    bool loss_on = false;          // rba_set_observation_loss, DESIGN.md section 21: the loss records = D.obs_loss while loss_on
    DeviceBuffer<S> loss;          // float [nslots] {scale, uint32 kind}; double [nslots] scale + [nslots] uint8 kind (loss_records)
  } obs;
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
  // linear_solver_type = DENSE_SCHUR (dense_solve.cuh, DESIGN.md section 27): the buffers of every solve, allocated by
  // setup_dense.  A: the np x np matrix and its factor; W, Tt: the potrf scratch; d: the scaling; x, y: the right-hand side
  // and the two substitutions; jp, kb: the per-slot rows; fail: the smallest failed pivot
  struct DenseSolve {
    double* A = nullptr; double* W = nullptr; double* Tt = nullptr; double* d = nullptr;
    double* x = nullptr; double* y = nullptr; double* jp = nullptr; double* kb = nullptr;
    int* fail = nullptr;
    long long np = 0;
  } dn;
  // preconditioner_type = CLUSTER_JACOBI (cluster_precond.cuh, DESIGN.md section 28).  The clustering's structure, blocks,
  // factors and statuses are the term's own (rba_set_camera_clusters adopts new ones once they all exist); bh (L^-1 b),
  // w (L^-T v), yh (L^-1 S w) and eye (the vector step's identity blocks) are allocated once by setup_clusters.
  struct ClusterTerm {
    bool on = false;
    std::vector<int> host, dflt;   // [nc] the clustering in use, the default one (rba_cluster_cameras at create)
    int ncl = 0, max_k = 0;
    long long blk_n = 0, fac_n = 0;  // doubles of the blocks and of the factors
    DeviceBuffer<int> ptr, cams, xb_ptr, status;
    DeviceBuffer<long long> blk_off, fac_off;
    DeviceBuffer<ClusterBlock> xb;
    DeviceBuffer<IntPair> slots;
    DeviceBuffer<AsmTerm> panel_terms;
    DeviceBuffer<double> blocks, factor;
    S* bh = nullptr; S* w = nullptr; S* yh = nullptr; S* eye = nullptr;
    bool built = false;            // a solve has assembled the blocks of this clustering
    void adopt(ClusterTerm& o) {
      ptr.take(o.ptr); cams.take(o.cams); xb_ptr.take(o.xb_ptr); status.take(o.status); blk_off.take(o.blk_off);
      fac_off.take(o.fac_off); xb.take(o.xb); slots.take(o.slots); panel_terms.take(o.panel_terms); blocks.take(o.blocks);
      factor.take(o.factor);
    }
  } clu;
  // assembled operator (setup_assembled, assembled.cuh): the terms as panel addresses in landmark-major order, the pair
  // list (term ranges, landmark-major position of every term), per pair its positions (lower, upper or -1) in the full
  // block-row CSR of S, the staging buffer of all terms, S_u per pair and S
  // asm_on: the structure exists; su_valid: S_u belongs to the current linearisation; s_valid: S = S_u + the damping part of
  // the last solve's lambda, and that solve (and rba_right_multiply / rba_time_matvec after it) applies S; su_new: this solve
  // enqueued the build of S_u (both reset when a solve starts)
  bool asm_on = false, su_valid = false, s_valid = false, su_new = false;
  int asm_nblk = 0, asm_switch = 0; long long asm_nt = 0, asm_nnzb = 0;
  AsmTerm* d_asm_terms = nullptr; int* d_asm_wpos = nullptr; int* d_asm_blk_ptr = nullptr; IntPair* d_asm_pos = nullptr;
  IntPair* d_asm_slots = nullptr;
  int* d_asm_col = nullptr;
  S* d_asm_stage = nullptr; S* d_asm_Su = nullptr; S* d_asm_S = nullptr;
  // k_rcs_spmv's deal (deal_spmv): its chunks, CTA by CTA, for spmv_grid co-resident CTAs
  SpmvChunk* d_spmv_chunks = nullptr; int* d_spmv_chunk_ptr = nullptr; int spmv_grid = 0, spmv_cap = 0;
  // s_fresh: the assembly has just been enqueued, so the next k_rcs_spmv must not read S before the assembly has completed:
  // it is a plain stream launch (its bulk copies of S start before griddepcontrol.wait, which orders only against the
  // kernel right before it, and k_rcs_mirror, the last writer of S, never triggers its dependents)
  bool s_fresh = false;

  ~Solver() override {
    if (comm && nccl) nccl->CommDestroy(comm);
    for (void* p : ipc_opened) cudaIpcCloseMemHandle(p);
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

  // Every device allocation of the handle: max(count, 1) entries, zeroed on the stream when asked; device_bytes counts all but
  // the covariance lists and per-call scratch (`counted` false) and never goes down (the most the handle has allocated).
  template <class T>
  int alloc(DeviceBuffer<T>& b, size_t count, bool zero, bool counted = true) {
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    void* q = nullptr;
    CU(cudaMalloc(&q, bytes));
    b = DeviceBuffer<T>((T*)q, count);
    if (counted) device_bytes += bytes;
    if (zero) CU(cudaMemsetAsync(q, 0, bytes, stream));
    return RBA_OK;
  }
  template <class T>
  int copy_in(T* dst, const std::vector<T>& v) {
    if (!v.empty()) CU(cudaMemcpyAsync(dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream));
    return RBA_OK;
  }
  // A buffer that lives as long as the handle (set-up), owned as max(count, 1) * sizeof(T) bytes.
  template <class T>
  int dalloc(T** p, size_t count, bool zero = true, bool counted = true) {
    DeviceBuffer<char> b;
    TRY(alloc(b, std::max<size_t>(count, 1) * sizeof(T), zero, counted));
    *p = (T*)b.get();
    owned.push_back(std::move(b));
    return RBA_OK;
  }
  template <class T>
  int upload(T** p, const std::vector<T>& v, bool counted = true) {
    TRY(dalloc(p, v.size(), false, counted));
    return copy_in(*p, v);
  }
  // A setter's buffer of `count` entries: the term's own `cur` while it holds as many, else a new one (not zeroed) in
  // `next`, which the setter adopts once every buffer of its call exists.  `src` is copied into the one chosen.
  template <class T>
  int fit(DeviceBuffer<T>& next, const DeviceBuffer<T>& cur, size_t count, const std::vector<T>* src = nullptr) {
    if (!cur.get() || cur.size() < count) TRY(alloc(next, count, false));
    return src ? copy_in(next.get() ? next.get() : cur.get(), *src) : RBA_OK;
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
    TRY(setup_dense());
    TRY(setup_clusters(pv));
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
    if (opt.linear_solver_type != 0 && opt.linear_solver_type != 1) { g_err = "linear_solver_type must be 0 (ITERATIVE_SCHUR) or 1 (DENSE_SCHUR)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.linear_solver_type == 1 && opt.solver_type == 2) { g_err = "DENSE_SCHUR does not combine with POWER_SCHUR_COMPLEMENT: the power series is itself the linear solver"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.linear_solver_type == 1 && opt.nranks > 1) { g_err = "DENSE_SCHUR runs on one GPU: the dense reduced camera matrix would need a cross-rank sum"; return RBA_ERR_UNSUPPORTED; }
    if (opt.preconditioner_type < 0 || opt.preconditioner_type > 2) { g_err = "preconditioner_type must be 0 (JACOBI), 1 (SCHUR_JACOBI) or 2 (CLUSTER_JACOBI)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.preconditioner_type == 2 && opt.solver_type == 2) { g_err = "CLUSTER_JACOBI does not combine with POWER_SCHUR_COMPLEMENT: the power series has no PCG"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.preconditioner_type == 2 && opt.linear_solver_type == 1) { g_err = "CLUSTER_JACOBI does not combine with DENSE_SCHUR: the dense solve has no PCG"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.preconditioner_type == 2 && opt.nranks > 1) { g_err = "CLUSTER_JACOBI runs on one GPU: a cluster block would need a cross-rank sum"; return RBA_ERR_UNSUPPORTED; }
    if (opt.stage2_form != 0 && opt.stage2_form != 1) { g_err = "stage2_form must be 0 (Q2 panel, reference) or 1 (orthogonality identity)"; return RBA_ERR_INVALID_ARGUMENT; }
    if (opt.pcg_check_period <= 0) opt.pcg_check_period = 4;
    if (opt.residual_reset_period <= 0) opt.residual_reset_period = 10;
    if (opt.power_order <= 0) opt.power_order = 20;  // solver_options.hpp:270
    // the Schur-complement solvers share the per-observation records and the implicit operator kernels (k_sc_stage2)
    panels = opt.operator_form == 0 && opt.solver_type == 0;
    ko.use_valid_projections_only = opt.use_valid_projections_only;
    ko.robust_norm = opt.robust_norm;
    ko.write_panel = panels;
    ko.huber = opt.huber_parameter;
    ko.jacobi_eps = opt.jacobi_scaling_epsilon > 0 ? opt.jacobi_scaling_epsilon : (double)ST<S>::eps_sqrt();  // ref: linearizor_base.cpp:72-79
    return RBA_OK;
  }
  // gradient and SCHUR_JACOBI blocks from the stored Q2 panels like the reference, instead of the orthogonality identities
  bool panel_form() const { return panels && opt.stage2_form == 0; }

  // Test hooks, not options: each forces at small size a path that the solver also takes on its own.
  //   RBA_PCG_PARTIALS=0  PCG without the per-segment hand-over to the vector kernel (taken above 1808 cameras)
  //   RBA_PCG_CLUSTER=k   a PCG vector cluster of at most k CTAs (taken when the device grants fewer than 16)
  //   RBA_PEER_AR=0       NCCL for the reductions across shards (taken when the IPC mapping of a peer fails)
  //   RBA_ASSEMBLED_RCS=0 the panel product P^T (P x) instead of the assembled S x (taken when S does not qualify)
  //   RBA_ASSEMBLED_AT=k  S built at PCG iteration k instead of the break-even iteration (taken by solves that run long)
  //   RBA_SPMV_CTAS=k     S x dealt over at most k CTAs (several rows and stage-ring wraps per CTA, taken by problems with
  //                       more block rows than co-resident CTAs)
  void read_test_hooks() {
    if (const char* e = getenv("RBA_PCG_PARTIALS")) pcg_partials = atoi(e) != 0;
    if (const char* e = getenv("RBA_PCG_CLUSTER")) pcg_cluster = std::max(1, std::min(atoi(e), 16));
    if (const char* e = getenv("RBA_PEER_AR")) peer_ar = atoi(e) != 0;
    if (const char* e = getenv("RBA_ASSEMBLED_RCS")) asm_hook = atoi(e) != 0;
    if (const char* e = getenv("RBA_ASSEMBLED_AT")) asm_at = std::max(0, atoi(e));
    if (const char* e = getenv("RBA_SPMV_CTAS")) spmv_cap = std::max(1, atoi(e));
  }

  int upload_layout(const rba_problem_view* pv) {
    nc = pv->num_cameras;
    nl_total = pv->num_landmarks;
    nobs_total = pv->lm_obs_offset[nl_total];
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
    if (panels) { op_slots = d_csr_y_slots; op_items = d_csr_y_items; op_item_ptr = d_csr_y_item_ptr; n_op_items = n_y_items; }
    else { op_slots = d_csr_obs_slots; op_items = d_csr_obs_items; op_item_ptr = d_csr_obs_item_ptr; n_op_items = n_obs_items; }
    TRY(upload(&d_pb_items, L.pb_items));
    TRY(upload(&d_pb_item_ptr, L.pb_cam_item_ptr));
    n_pb_items = (int)L.pb_items.size();
    return RBA_OK;
  }

  // The grids of the persistent kernels and the order in which their warps take the work.
  int deal_work() {
    if (panels) {
      TRY(deal_matvec_items());
    } else {
      while (imp_tile_split < (int)L.tiles.size() && (32 / L.tiles[imp_tile_split].G) * L.tiles[imp_tile_split].n <= IMP_MAXSLOTS) ++imp_tile_split;
      imp_smem = (size_t)IMP_WARPS * IMP_NS * (size_t)IMP_MAXSLOTS * 48 * sizeof(S);
      CU(cudaFuncSetAttribute((k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)imp_smem));
      int bps = 0;
      CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, (k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), IMP_WARPS * 32, imp_smem));
      imp_grid = std::max(1, std::min((imp_tile_split + IMP_WARPS - 1) / IMP_WARPS, sm_count * std::max(1, bps)));
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
    if (panels) TRY(dalloc(&D.panel, (size_t)L.panel_scalars));
    TRY(dalloc(&D.jp, (size_t)20 * L.nslots));
    TRY(dalloc(&D.q1u, (size_t)28 * L.nslots));
    TRY(dalloc(&D.q1d, (size_t)28 * L.nslots));
    TRY(dalloc(&D.jl, (size_t)6 * L.nslots));
    TRY(dalloc(&D.res, (size_t)2 * L.nslots));
    TRY(dalloc(&D.lmk, (size_t)24 * L.sorted_lm.size()));
    TRY(dalloc(&D.qtr, (size_t)2 * L.nslots));
    // the damping rows per slot: read by the SCHUR_JACOBI blocks of the panel form and by the assembly of S
    if (panel_form() || asm_candidate()) TRY(dalloc(&D.dmp, (size_t)28 * L.nslots));
    if (panel_form()) {
      if (opt.preconditioner_type >= 1) TRY(dalloc(&D.blk0, (size_t)48 * L.nslots));  // (CLUSTER_JACOBI: its diagonal blocks)
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

  // The per-observation instances of the kernels that evaluate the reprojection terms: OBSW with observation information
  // (D.obs_W, section 19), OBSL with observation losses (D.obs_loss, section 21); both off = the unmodified kernels
  static auto k_error_instance(bool obsw, bool obsl) {
    return obsw ? (obsl ? k_error<S, true, true> : k_error<S, true>) : (obsl ? k_error<S, false, true> : k_error<S>);
  }
  static auto k_jp_norms_instance(bool obsw, bool obsl) {
    return obsw ? (obsl ? k_jp_norms<S, true, true> : k_jp_norms<S, true>) : (obsl ? k_jp_norms<S, false, true> : k_jp_norms<S>);
  }
  template <bool GIVENS, bool LMP>
  static auto k1_of(bool obsw, bool obsl) {
    return obsw ? (obsl ? k_linearize_qr<S, GIVENS, LMP, true, true> : k_linearize_qr<S, GIVENS, LMP, true>)
                : (obsl ? k_linearize_qr<S, GIVENS, LMP, false, true> : k_linearize_qr<S, GIVENS, LMP>);
  }
  static auto k1_instance(bool givens, bool lmp, bool obsw, bool obsl) {  // + LMP: the landmark priors (section 17)
    return givens ? (lmp ? k1_of<true, true>(obsw, obsl) : k1_of<true, false>(obsw, obsl))
                  : (lmp ? k1_of<false, true>(obsw, obsl) : k1_of<false, false>(obsw, obsl));
  }
  template <bool LMP>
  static auto kcov_of(bool obsw, bool obsl) {
    return obsw ? (obsl ? k_cov_landmark<S, LMP, true, true> : k_cov_landmark<S, LMP, true>)
                : (obsl ? k_cov_landmark<S, LMP, false, true> : k_cov_landmark<S, LMP>);
  }
  static auto kcov_lmpl(bool obsw, bool obsl) {  // + LMPL: the landmark priors' losses (section 22)
    return obsw ? (obsl ? k_cov_landmark<S, true, true, true, true> : k_cov_landmark<S, true, true, false, true>)
                : (obsl ? k_cov_landmark<S, true, false, true, true> : k_cov_landmark<S, true, false, false, true>);
  }

  int setup_kernels() {
    if (k1_sc.gstride) TRY(dalloc(&k1_sc.gbase, (size_t)(k1_max_blocks * TILE_WARPS) * k1_sc.gstride, false));
    if (k2_sc.gstride) TRY(dalloc(&k2_sc.gbase, (size_t)(k2_max_blocks * TILE_WARPS) * k2_sc.gstride, false));
    // every k_linearize_qr instance: both QR variants, with and without landmark priors (section 17), observation
    // information (section 19) and observation losses (section 21)
    for (int v = 0; v < 16; ++v)
      CU(cudaFuncSetAttribute(k1_instance(v & 8, v & 4, v & 2, v & 1), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
    CU(cudaFuncSetAttribute((k_stage2<S, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));
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
    std::vector<S> tied;
    if (grp.n) {  // the members take their lead's f, k1, k2
      tied.assign((const S*)cams, (const S*)cams + (size_t)10 * nc);
      tie_intrinsics(tied.data());
      cams = tied.data();
    }
    CU(cudaMemcpyAsync(D.cams, cams, (size_t)10 * nc * sizeof(S), cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(D.lms, (const S*)lms + (size_t)3 * L.lm_begin, (size_t)3 * L.nl_local * sizeof(S), cudaMemcpyHostToDevice, stream));
    if (rig.n) TRY(rig_retie_state(D.cams));  // the members take M_j T_lead
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
    std::vector<uint8_t> fl;
    if (any) fl.assign(flags, flags + nc);
    if (grp.n) {
      const std::string why = group_flags_mismatch(grp.host_lead, fl);
      if (!why.empty()) { g_err = "rba_set_camera_fixed: " + why; return RBA_ERR_INVALID_ARGUMENT; }
    }
    if (rig.n) {
      const std::string why = rig_flags_mismatch(rig.host_lead, fl);
      if (!why.empty()) { g_err = "rba_set_camera_fixed: " + why; return RBA_ERR_INVALID_ARGUMENT; }
    }
    if (any) {
      DeviceBuffer<uint8_t> next; TRY(fit(next, held.flags, (size_t)nc, &fl));
      CU(cudaStreamSynchronize(stream));
      held.flags.take(next);
    }
    held.all = all;
    held.host = std::move(fl);
    point_at_terms();
    TRY(upload_tied_fixed());
    have_inc = false;  // the device-resident increment was solved under the previous flags
    return RBA_OK;
  }

  // Intrinsics shared across groups of cameras (DESIGN.md section 18).  Every check runs before anything changes, so a
  // rejected call leaves the previous groups.  No group of >= 2 cameras = the unmodified path (grp.n == 0).
  int set_intrinsics_groups(const int32_t* group) override {
    auto fail = [&](int rc, const std::string& what) { g_err = "rba_set_intrinsics_groups: " + what; return rc; };
    std::vector<int> lead((size_t)nc, -1), first((size_t)nc, -1), count((size_t)nc, 0);
    if (group) {
      for (int c = 0; c < nc; ++c) {
        const int g = group[c];
        if (g < -1 || g >= nc)
          return fail(RBA_ERR_INVALID_ARGUMENT, "camera " + std::to_string(c) + " has group id " + std::to_string(g) + ", outside [-1, " + std::to_string(nc) + ")");
        if (g >= 0 && count[g]++ == 0) first[g] = c;
      }
      for (int c = 0; c < nc; ++c)
        if (group[c] >= 0 && count[group[c]] >= 2) lead[c] = first[group[c]];
    }
    // groups in the order of their leads, members ascending (the lead first)
    std::vector<int> gidx((size_t)nc, -1), ptr(1, 0), mem;
    int ng = 0;
    for (int c = 0; c < nc; ++c)
      if (lead[c] == c) gidx[c] = ng++;
    if (ng > 0 && opt.solver_type == 2)
      return fail(RBA_ERR_UNSUPPORTED, "POWER_SCHUR_COMPLEMENT does not support groups of >= 2 cameras (Hpp of the tied problem is not block-diagonal)");
    if (ng > 0 && clu.on)
      return fail(RBA_ERR_UNSUPPORTED, "CLUSTER_JACOBI does not support groups of >= 2 cameras (the tied system changes the unknowns of the cluster blocks)");
    const std::string why = group_flags_mismatch(lead, held.host);
    if (!why.empty()) return fail(RBA_ERR_INVALID_ARGUMENT, why);
    ptr.assign((size_t)ng + 1, 0);
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0) ++ptr[gidx[lead[c]] + 1];
    for (int g = 0; g < ng; ++g) ptr[g + 1] += ptr[g];
    mem.resize((size_t)ptr[ng]);
    std::vector<int> fill(ptr.begin(), ptr.end() - 1);
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0) mem[fill[gidx[lead[c]]]++] = c;
    if (ng > 0) {
      GroupTerm next;
      TRY(fit(next.lead, {}, lead.size(), &lead)); TRY(fit(next.ptr, {}, ptr.size(), &ptr)); TRY(fit(next.mem, {}, mem.size(), &mem));
      if (!grp.ve.get()) { TRY(alloc(next.ve, (size_t)9 * nc, true)); TRY(alloc(next.y, (size_t)9 * nc, true)); TRY(alloc(next.fixed, (size_t)nc, true)); }
      CU(cudaStreamSynchronize(stream));
      grp.adopt(next);
    }
    grp.n = ng;
    grp.host_lead = std::move(lead);
    TRY(upload_tied_fixed());
    if (ng > 0) {
      // the current state and its backup take the tied values
      std::vector<S> c((size_t)10 * nc);
      for (S* d : std::initializer_list<S*>{D.cams, cams_bk}) {
        CU(cudaMemcpyAsync(c.data(), d, c.size() * sizeof(S), cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        tie_intrinsics(c.data());
        CU(cudaMemcpyAsync(d, c.data(), c.size() * sizeof(S), cudaMemcpyHostToDevice, stream));
      }
      CU(cudaStreamSynchronize(stream));
      ++state_version;
    }
    // the scaling, b and the blocks of the last linearisation belong to the previous groups
    return priors_changed();
  }
  // "" when every group's members agree on RBA_FIX_F / K1 / K2, else which camera does not
  std::string group_flags_mismatch(const std::vector<int>& lead, const std::vector<uint8_t>& flags) const {
    if (flags.empty()) return "";
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0 && (flags[c] & RBA_FIX_INTRINSICS) != (flags[lead[c]] & RBA_FIX_INTRINSICS))
        return "camera " + std::to_string(c) + " has RBA_FIX_F / K1 / K2 bits " + std::to_string(flags[c] & RBA_FIX_INTRINSICS) +
               " that differ from those of its group's lead, camera " + std::to_string(lead[c]) + " (" + std::to_string(flags[lead[c]] & RBA_FIX_INTRINSICS) + ")";
    return "";
  }
  void tie_intrinsics(S* cams) const {
    for (int c = 0; c < nc; ++c)
      if (grp.host_lead[c] >= 0 && grp.host_lead[c] != c)
        for (int k = 7; k < 10; ++k) cams[10 * (size_t)c + k] = cams[10 * (size_t)grp.host_lead[c] + k];
  }
  // the flags k_precond_invert masks with while groups or rigs exist (grp.fixed, rig.fixed): the user's, the intrinsics of
  // every group member but the lead and the pose of every rig member but the lead.  With sensors (section 24) a home's pose
  // entries carry its sensor's, which RBA_FIX_POSE on its rig does not hold; the camera update and the other users of
  // D.cam_fixed then read the user's flags without RBA_FIX_POSE on the sensor cameras (sen.cam_fixed).
  int upload_tied_fixed() {
    if (!grp.n && !rig.n) return RBA_OK;
    std::vector<uint8_t> f((size_t)nc, 0);
    auto member = [](const std::vector<int>& lead, int c) { return !lead.empty() && lead[c] >= 0 && lead[c] != c; };
    for (int c = 0; c < nc; ++c)
      f[c] = (uint8_t)((held.host.empty() ? 0 : held.host[c]) | (grp.n && member(grp.host_lead, c) ? RBA_FIX_INTRINSICS : 0) |
                       (rig.n && member(rig.host_lead, c) ? RBA_FIX_POSE : 0));
    if (sen.n) {
      std::vector<uint8_t> user((size_t)nc, 0);
      for (int c = 0; c < nc; ++c)
        if (sen.host_home[c] >= 0) {
          if (sen.host_home[c] == c) f[c] &= (uint8_t)~RBA_FIX_POSE;
          if (!held.host.empty()) user[c] = (uint8_t)(held.host[c] & ~RBA_FIX_POSE);
        } else if (!held.host.empty()) {
          user[c] = held.host[c];
        }
      if (!held.host.empty()) TRY(copy_in(sen.cam_fixed.get(), user));
    }
    if (grp.n) TRY(copy_in(grp.fixed.get(), f));
    if (rig.n) TRY(copy_in(rig.fixed.get(), f));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }
  const uint8_t* tied_fixed() const { return rig.n ? rig.fixed.get() : grp.fixed.get(); }
  GroupView groups() const { return {grp.lead.get(), grp.ptr.get(), grp.mem.get(), grp.n}; }
  int group_expand(const S* v, S* out, bool in_solve) {
    return launch_ex(k_group_expand<S>, (9 * nc + 255) / 256, 256, 0, in_solve, 1, v, out, (const int*)grp.lead.get(), nc,
                     in_solve ? (const PcgState*)d_state : (const PcgState*)nullptr);
  }
  // Rigid camera rigs (DESIGN.md section 23).  Every check runs before anything changes, and the new buffers are adopted
  // once they all exist, so a rejected call leaves the previous rigs.  No rig of >= 2 cameras = the unmodified path (rig.n
  // == 0).
  int set_camera_rigs(const int32_t* rid, const void* cam_from_rig) override {
    auto fail = [&](int rc, const std::string& what) { g_err = "rba_set_camera_rigs: " + what; return rc; };
    if (!rid != !cam_from_rig) return fail(RBA_ERR_INVALID_ARGUMENT, "rig and cam_from_rig must both be given or both be NULL");
    std::vector<int> lead((size_t)nc, -1), first((size_t)nc, -1), count((size_t)nc, 0);
    std::vector<double> E((size_t)7 * nc, 0.0);  // the extrinsics of every rigged camera, quaternion normalised
    if (rid) {
      const S* e = (const S*)cam_from_rig;
      for (int c = 0; c < nc; ++c) {
        const int r = rid[c];
        if (r < -1 || r >= nc)
          return fail(RBA_ERR_INVALID_ARGUMENT, "camera " + std::to_string(c) + " has rig id " + std::to_string(r) + ", outside [-1, " + std::to_string(nc) + ")");
        if (r < 0) continue;
        if (count[r]++ == 0) first[r] = c;
        double qn = 0;
        for (int k = 0; k < 7; ++k) {
          const double v = (double)e[7 * (size_t)c + k];
          if (!std::isfinite(v)) return fail(RBA_ERR_INVALID_ARGUMENT, "camera " + std::to_string(c) + " has a non-finite cam_from_rig");
          E[7 * (size_t)c + k] = v;
          if (k < 4) qn += v * v;
        }
        qn = std::sqrt(qn);
        if (!(std::fabs(qn - 1.0) <= 1e-3))
          return fail(RBA_ERR_INVALID_ARGUMENT, "camera " + std::to_string(c) + " has a cam_from_rig quaternion of norm " + std::to_string(qn) + " (must be within 1e-3 of 1)");
        for (int k = 0; k < 4; ++k) E[7 * (size_t)c + k] /= qn;
      }
      for (int c = 0; c < nc; ++c)
        if (rid[c] >= 0 && count[rid[c]] >= 2) lead[c] = first[rid[c]];
    }
    int nr = 0;
    for (int c = 0; c < nc; ++c) nr += lead[c] == c;
    if (nr > 0 && opt.solver_type == 2)
      return fail(RBA_ERR_UNSUPPORTED, "POWER_SCHUR_COMPLEMENT does not support rigs of >= 2 cameras (Hpp of the tied problem is not block-diagonal)");
    if (nr > 0 && clu.on)
      return fail(RBA_ERR_UNSUPPORTED, "CLUSTER_JACOBI does not support rigs of >= 2 cameras (the tied system changes the unknowns of the cluster blocks)");
    const std::string why = rig_flags_mismatch(lead, held.host);
    if (!why.empty()) return fail(RBA_ERR_INVALID_ARGUMENT, why);
    if (nr > 0) {
      RigTerm next;
      TRY(rig_tables(lead, E, {}, next, nullptr));
      CU(cudaStreamSynchronize(stream));
      rig.adopt(next);
    }
    rig.n = nr;
    rig.host_first = lead;
    rig.host_lead = std::move(lead);
    rig.host_E = std::move(E);
    sen.n = 0;  // the sensors belonged to the previous rigs
    sen.host_home.clear();
    TRY(upload_tied_fixed());
    if (nr > 0) {  // the current state and its backup take the tied poses
      TRY(rig_retie(D.cams)); TRY(rig_retie(cams_bk));
      CU(cudaStreamSynchronize(stream));
      ++state_version;
    }
    // the blocks and b of the last linearisation belong to the previous rigs
    return priors_changed();
  }
  // m = a b^-1 of two poses (qx,qy,qz,qw, tx,ty,tz) in double, the quaternion normalised
  static void pose_ratio(const double* a, const double* l, double* m) {
    const double b0 = -l[0], b1 = -l[1], b2 = -l[2], b3 = l[3];
    m[3] = a[3] * b3 - a[0] * b0 - a[1] * b1 - a[2] * b2;
    m[0] = a[3] * b0 + a[0] * b3 + a[1] * b2 - a[2] * b1;
    m[1] = a[3] * b1 + a[1] * b3 + a[2] * b0 - a[0] * b2;
    m[2] = a[3] * b2 + a[2] * b3 + a[0] * b1 - a[1] * b0;
    const double qn = std::sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2] + m[3] * m[3]);
    for (int k = 0; k < 4; ++k) m[k] /= qn;
    const double R[9] = {1 - 2 * (m[1] * m[1] + m[2] * m[2]), 2 * (m[0] * m[1] - m[2] * m[3]), 2 * (m[0] * m[2] + m[1] * m[3]),
                         2 * (m[0] * m[1] + m[2] * m[3]), 1 - 2 * (m[0] * m[0] + m[2] * m[2]), 2 * (m[1] * m[2] - m[0] * m[3]),
                         2 * (m[0] * m[2] - m[1] * m[3]), 2 * (m[1] * m[2] + m[0] * m[3]), 1 - 2 * (m[0] * m[0] + m[1] * m[1])};
    for (int r = 0; r < 3; ++r) m[4 + r] = a[4 + r] - (R[3 * r] * l[4] + R[3 * r + 1] * l[5] + R[3 * r + 2] * l[6]);
  }
  // The device tables of the rigs whose cameras have the leads `lead` (>= 1 rig of >= 2 cameras) and the extrinsics E, into
  // next: the rigs in the order of their leads, each one's members with the lead first and the others ascending;
  // M_j = E_j E_lead^-1 and its adjoint A_j = [[R_M, [t_M]x R_M], [0, R_M]] (the identity for a lead).  With sensors (home
  // not empty) a sensor camera j takes M_j = E_home E_lead^-1 (the call ties it to its home's extrinsics) and
  // K_j = E_lead(home) E_lead^-1 goes into *K.
  int rig_tables(const std::vector<int>& lead, const std::vector<double>& E, const std::vector<int>& home, RigTerm& next,
                 std::vector<double>* K) {
    std::vector<int> ridx((size_t)nc, -1), ptr(1, 0), mem;
    int nr = 0;
    for (int c = 0; c < nc; ++c)
      if (lead[c] == c) ridx[c] = nr++;
    ptr.assign((size_t)nr + 1, 0);
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0) ++ptr[ridx[lead[c]] + 1];
    for (int r = 0; r < nr; ++r) ptr[r + 1] += ptr[r];
    mem.resize((size_t)ptr[nr]);
    std::vector<int> fill(ptr.begin(), ptr.end() - 1);
    for (int c = 0; c < nc; ++c)
      if (lead[c] == c) mem[fill[ridx[c]]++] = c;
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0 && lead[c] != c) mem[fill[ridx[lead[c]]]++] = c;
    std::vector<double> M((size_t)7 * nc, 0.0);
    std::vector<S> adj((size_t)36 * nc, S(0));
    if (K) K->assign((size_t)7 * nc, 0.0);
    for (int c = 0; c < nc; ++c) {
      if (lead[c] < 0) continue;
      const int src = home.empty() || home[c] < 0 ? c : home[c];
      double* m = &M[7 * (size_t)c];
      pose_ratio(&E[7 * (size_t)src], &E[7 * (size_t)lead[c]], m);
      if (src != c) pose_ratio(&E[7 * (size_t)lead[src]], &E[7 * (size_t)lead[c]], &(*K)[7 * (size_t)c]);
      if (K && src == c && !home.empty() && home[c] == c) (*K)[7 * (size_t)c + 3] = 1.0;
      const double x = m[0], y = m[1], z = m[2], w = m[3];
      const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                           2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                           2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
      const double tx[9] = {0, -m[6], m[5], m[6], 0, -m[4], -m[5], m[4], 0};
      S* A = &adj[36 * (size_t)c];
      for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) {
          double txr = 0;
          for (int i = 0; i < 3; ++i) txr += tx[3 * r + i] * R[3 * i + k];
          A[6 * r + k] = (S)R[3 * r + k];
          A[6 * r + 3 + k] = (S)txr;
          A[6 * (3 + r) + 3 + k] = (S)R[3 * r + k];
        }
      if (c == lead[c])  // exactly the identity
        for (int k = 0; k < 36; ++k) A[k] = (k % 7 == 0) ? S(1) : S(0);
    }
    TRY(fit(next.lead, {}, lead.size(), &lead)); TRY(fit(next.ptr, {}, ptr.size(), &ptr)); TRY(fit(next.mem, {}, mem.size(), &mem));
    TRY(fit(next.adj, {}, adj.size(), &adj)); TRY(fit(next.M, {}, M.size(), &M));
    TRY(fit(next.du, rig.du, (size_t)6 * nr));
    if (!rig.ve.get()) {
      TRY(alloc(next.pt, (size_t)36 * nc, true)); TRY(alloc(next.fixed, (size_t)nc, true));
      TRY(alloc(next.ve, (size_t)9 * nc, true)); TRY(alloc(next.y, (size_t)9 * nc, true));
    }
    return RBA_OK;
  }
  // Estimated extrinsics shared by the captures of one sensor (DESIGN.md section 24).  Every check runs before anything
  // changes and the new buffers are adopted once they all exist, so a rejected or failed call leaves the previous sensors.
  // No sensor id = the rigs of section 23 (sen.n == 0), their lead the lowest-index camera again.
  int set_rig_sensors(const int32_t* sensor) override {
    auto fail = [&](const std::string& what) { g_err = "rba_set_rig_sensors: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    std::vector<int> home((size_t)nc, -1), lead = rig.host_first;
    int ns = 0;
    if (sensor && clu.on && std::any_of(sensor, sensor + nc, [](int32_t v) { return v >= 0; })) {
      g_err = "rba_set_rig_sensors: CLUSTER_JACOBI does not support sensors (the tied system changes the unknowns of the cluster blocks)";
      return RBA_ERR_UNSUPPORTED;
    }
    if (sensor) {
      std::vector<int> first((size_t)nc, -1), new_lead((size_t)nc, -1);
      std::vector<std::pair<int, int>> rig_sensor;  // (the rig's lowest-index camera, sensor id) of every sensor camera
      for (int c = 0; c < nc; ++c) {
        const int sid = sensor[c];
        if (sid < -1 || sid >= nc)
          return fail("camera " + std::to_string(c) + " has sensor id " + std::to_string(sid) + ", outside [-1, " + std::to_string(nc) + ")");
        if (sid < 0) {
          if (rig.n && rig.host_first[c] >= 0 && new_lead[rig.host_first[c]] < 0) new_lead[rig.host_first[c]] = c;
          continue;
        }
        if (!rig.n || rig.host_first[c] < 0)
          return fail("camera " + std::to_string(c) + " has sensor id " + std::to_string(sid) + " but is not in a rig of >= 2 cameras");
        if (first[sid] < 0) { first[sid] = c; ++ns; }
        home[c] = first[sid];
        rig_sensor.push_back({rig.host_first[c], sid});
      }
      std::sort(rig_sensor.begin(), rig_sensor.end());
      for (size_t k = 1; k < rig_sensor.size(); ++k)
        if (rig_sensor[k] == rig_sensor[k - 1])
          return fail("two cameras of the rig led by camera " + std::to_string(rig_sensor[k].first) + " have sensor id " + std::to_string(rig_sensor[k].second));
      for (int c = 0; c < nc; ++c)
        if (rig.n && rig.host_first[c] == c && new_lead[c] < 0)
          return fail("every camera of the rig led by camera " + std::to_string(c) + " has a sensor id: none is left to carry the rig's pose");
      for (int c = 0; c < nc; ++c)
        if (rig.n && rig.host_first[c] >= 0) lead[c] = new_lead[rig.host_first[c]];
    }
    if (!rig.n) {  // nothing to tie, nothing to clear
      sen.n = 0;
      return RBA_OK;
    }
    // the sensors in the order of their homes, each one's cameras ascending (the home first)
    std::vector<int> sidx((size_t)nc, -1), sptr((size_t)ns + 1, 0), smem;
    for (int c = 0, k = 0; c < nc; ++c)
      if (home[c] == c) sidx[c] = k++;
    for (int c = 0; c < nc; ++c)
      if (home[c] >= 0) ++sptr[sidx[home[c]] + 1];
    for (int k = 0; k < ns; ++k) sptr[k + 1] += sptr[k];
    smem.resize((size_t)sptr[ns]);
    std::vector<int> fill(sptr.begin(), sptr.end() - 1);
    for (int c = 0; c < nc; ++c)
      if (home[c] >= 0) smem[fill[sidx[home[c]]]++] = c;
    RigTerm next;
    SensorTerm snext;
    std::vector<double> K;
    TRY(rig_tables(lead, rig.host_E, ns ? home : std::vector<int>{}, next, ns ? &K : nullptr));
    if (ns) {
      TRY(fit(snext.home, {}, home.size(), &home)); TRY(fit(snext.ptr, {}, sptr.size(), &sptr)); TRY(fit(snext.mem, {}, smem.size(), &smem));
      TRY(fit(snext.K, {}, K.size(), &K));
      TRY(fit(snext.qt, sen.qt, (size_t)6 * nc)); TRY(fit(snext.ds, sen.ds, (size_t)6 * ns));
      TRY(fit(snext.cam_fixed, sen.cam_fixed, (size_t)nc));
      TRY(fit(snext.blk, sen.blk, (size_t)81 * nc)); TRY(fit(snext.b, sen.b, (size_t)9 * nc));
    }
    CU(cudaStreamSynchronize(stream));
    rig.adopt(next);
    sen.adopt(snext);
    rig.host_lead = std::move(lead);
    sen.n = ns;
    sen.host_home = ns ? std::move(home) : std::vector<int>{};
    point_at_terms();
    TRY(upload_tied_fixed());
    // every member re-tied from its lead: the held ones through their extrinsics, a sensor's cameras through its home's
    TRY(rig_retie(D.cams)); TRY(rig_retie(cams_bk));
    CU(cudaStreamSynchronize(stream));
    ++state_version;
    return priors_changed();
  }
  // The extrinsics of every camera in the convention of rba_set_camera_rigs: held ones as given (normalised), a sensor's
  // E_s = T_home T_lead(home)^-1 E_lead(home) from the current state, free cameras the identity
  int get_rig_extrinsics(void* out) override {
    if (!out) { g_err = "rba_get_rig_extrinsics: cam_from_rig is NULL"; return RBA_ERR_INVALID_ARGUMENT; }
    std::vector<S> cams((size_t)10 * nc);
    CU(cudaMemcpyAsync(cams.data(), D.cams, cams.size() * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    S* o = (S*)out;
    auto pose = [&](int c, double* p) { for (int k = 0; k < 7; ++k) p[k] = (double)cams[10 * (size_t)c + k]; };
    for (int c = 0; c < nc; ++c) {
      double e[7] = {0, 0, 0, 1, 0, 0, 0};
      if (rig.n && rig.host_lead[c] >= 0) {
        const int h = sen.n ? sen.host_home[c] : -1;
        if (h < 0) {
          for (int k = 0; k < 7; ++k) e[k] = rig.host_E[7 * (size_t)c + k];
        } else {  // (T_home T_lead^-1) (E_lead^-1)^-1
          const int l = rig.host_lead[h];
          const double* el = &rig.host_E[7 * (size_t)l];
          double th[7], tl[7], x[7], one[7] = {0, 0, 0, 1, 0, 0, 0}, ei[7];
          pose(h, th); pose(l, tl);
          pose_ratio(th, tl, x);
          pose_ratio(one, el, ei);
          pose_ratio(x, ei, e);
        }
      }
      for (int k = 0; k < 7; ++k) o[7 * (size_t)c + k] = (S)e[k];
    }
    return RBA_OK;
  }
  // "" when every rig's members agree on RBA_FIX_POSE, else which camera does not
  std::string rig_flags_mismatch(const std::vector<int>& lead, const std::vector<uint8_t>& flags) const {
    if (flags.empty()) return "";
    for (int c = 0; c < nc; ++c)
      if (lead[c] >= 0 && (flags[c] & RBA_FIX_POSE) != (flags[lead[c]] & RBA_FIX_POSE))
        return "camera " + std::to_string(c) + " has the RBA_FIX_POSE bit " + std::to_string(flags[c] & RBA_FIX_POSE) +
               " that differs from that of its rig's lead, camera " + std::to_string(lead[c]) + " (" + std::to_string(flags[lead[c]] & RBA_FIX_POSE) + ")";
    return "";
  }
  RigView<S> rigs() const {
    return {rig.lead.get(), rig.ptr.get(), rig.mem.get(), rig.adj.get(), rig.M.get(), rig.pt.get(), rig.du.get(), rig.n};
  }
  SensorView<S> sensors() const {
    return {sen.home.get(), sen.ptr.get(), sen.mem.get(), sen.K.get(), sen.qt.get(), sen.ds.get(), sen.b.get(), rig.fixed.get(), sen.n};
  }
  int rig_ncb() const { return (nc + GROUP_THREADS - 1) / GROUP_THREADS; }
  // every member at M_j T_lead through the stored M_j (at the setters' calls, and always without sensors)
  int rig_retie(S* cams) {
    k_rig_retie<S><<<(nc + 127) / 128, 128, 0, stream>>>(cams, rigs(), nc);
    ++launches;
    return RBA_OK;
  }
  // after a camera update or rba_set_state: with sensors their cameras follow their homes (k_sensor_retie)
  int rig_retie_state(S* cams) {
    if (!sen.n) return rig_retie(cams);
    k_sensor_retie<S><<<(nc + 127) / 128, 128, 0, stream>>>(cams, rigs(), sensors(), nc);
    ++launches;
    return RBA_OK;
  }
  // M_j and A_j of the sensor cameras at the current state
  int sensor_tie() {
    k_sensor_tie<S><<<(nc + 127) / 128, 128, 0, stream>>>(D.cams, rigs(), sensors(), rig.M.get(), rig.adj.get(), nc);
    ++launches;
    return RBA_OK;
  }
  int rig_expand(const S* v, S* out, bool in_solve, int host = 0) {
    const PcgState* st = in_solve ? (const PcgState*)d_state : (const PcgState*)nullptr;
    if (sen.n)
      return launch_ex(k_rig_expand<S, true>, rig_ncb() + rig.n, GROUP_THREADS, 0, in_solve, 1, v, out, rigs(), nc, rig_ncb(), host, st,
                       sensors());
    return launch_ex(k_rig_expand<S>, rig_ncb() + rig.n, GROUP_THREADS, 0, in_solve, 1, v, out, rigs(), nc, rig_ncb(), host, st,
                     NoSensors{});
  }
  // the contracted operator output the vector step reads: the groups' unless rigs contract out of place (sensors)
  S* tied_y() const { return grp.n && !sen.n ? grp.y.get() : rig.y.get(); }
  // inc = P~ u (and P u of the groups) for the back-substitution, the update and inc_out (with sensors out of place: the
  // homes' entries are read across rigs)
  int tie_expand(S* inc) {
    if (rig.n && sen.n) {
      CU(cudaMemcpyAsync(rig.ve.get(), inc, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToDevice, stream));
      TRY(rig_expand(rig.ve.get(), inc, false));
    } else if (rig.n) {
      TRY(rig_expand(inc, inc, false));
    }
    if (grp.n) TRY(group_expand(inc, inc, false));
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
      CameraPriorTerm next;
      TRY(fit(next.mean, cprior.mean, (size_t)10 * nc, &mean)); TRY(fit(next.L, cprior.L, (size_t)81 * nc, &Lsq));
      TRY(fit(next.A, cprior.A, (size_t)81 * nc)); TRY(fit(next.r, cprior.r, (size_t)9 * nc));
      TRY(fit(next.H, cprior.H, (size_t)81 * nc)); TRY(fit(next.g, cprior.g, (size_t)9 * nc));
      CU(cudaStreamSynchronize(stream));
      cprior.adopt(next);
    }
    cprior.on = any;
    cprior.loss.on = false;
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
  CameraPrior<S> camera_prior() const { return {D.cams, cprior.mean.get(), cprior.L.get(), cprior.A.get(), cprior.r.get()}; }
  PairPrior<S> pair_prior() const { return {D.cams, pprior.ij.get(), pprior.mean.get(), pprior.L.get(), pprior.A.get(), pprior.r.get()}; }
  LandmarkPrior<S> landmark_prior() const { return {D.lms, lprior.lm.get(), lprior.mean.get(), lprior.L.get()}; }
  // The cost of the n items of one prior kind into the error sums (k_prior_cost): rho(s)/2 of their losses while `loss` is on
  // (section 22), else 1/2 s
  template <class K>
  int prior_cost(K k, int n, const PriorLoss& loss) {
    if (loss.on) k_prior_cost<<<1, 256, 0, stream>>>(RobustPrior<K>{k, loss.rec.get(), n}, n, d_red, d_flags);
    else k_prior_cost<<<1, 256, 0, stream>>>(k, n, d_red, d_flags);
    ++launches;
    return RBA_OK;
  }
  // Before the kernels of a linearisation read a prior kind's L: sqrt(w) L into loss.Lw while its losses are on (section 22).
  // Returns the L those kernels read.
  template <class K>
  const S* weighted_L(K k, int n, PriorLoss& loss) {
    if (!loss.on) return k.L;
    k_prior_weight<<<(n + 127) / 128, 128, 0, stream>>>(RobustPrior<K>{k, loss.rec.get(), n}, loss.Lw.get());
    ++launches;
    return loss.Lw.get();
  }
  // The kernels' optional pointers, from the problem terms (nullptr = the kernels without the term)
  void point_at_terms() {
    D.cam_fixed = held.host.empty() ? nullptr : sen.n ? sen.cam_fixed.get() : held.flags.get();
    D.prior_H = cprior.on || pprior.n > 0 ? cprior.H.get() : nullptr;
    D.pair_ptr = pprior.ptr.get(); D.pair_nbr = pprior.nbr.get(); D.pair_O = pprior.O.get();
    D.pair_ov = pprior.n > 0 ? pprior.ov.get() : nullptr;
    D.lmp_slot = lprior.n > 0 ? lprior.slot.get() : nullptr;
    D.lmp_mean = lprior.mean.get(); D.lmp_Lg = lprior.Lg.get();
    // losses on the landmark priors (section 22): the kernels that read L take sqrt(w) L
    D.lmp_L = lprior.loss.on ? lprior.loss.Lw.get() : lprior.L.get();
    D.lmp_Lu = lprior.L.get(); D.lmp_loss = lprior.loss.on ? lprior.loss.rec.get() : nullptr; D.lmp_n = lprior.n;
    D.obs_W = obs.on ? obs.W.get() : nullptr;
    D.obs_loss = obs.loss_on ? obs.loss.get() : nullptr;
  }
  int priors_changed() {
    point_at_terms();
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
    std::vector<int> ij, item_of((size_t)std::max(num_pairs, 0), -1);
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
      item_of[p] = (int)(ij.size() / 2);
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
      PairPriorTerm next; CameraPriorTerm diag;  // diag: H and g
      TRY(fit(next.ij, pprior.ij, 2 * (size_t)np, &ij)); TRY(fit(next.mean, pprior.mean, 7 * (size_t)np, &mean));
      TRY(fit(next.L, pprior.L, 36 * (size_t)np, &Lsq)); TRY(fit(next.A, pprior.A, 72 * (size_t)np));
      TRY(fit(next.r, pprior.r, 6 * (size_t)np)); TRY(fit(next.item, pprior.item, 2 * (size_t)np, &item));
      TRY(fit(next.nbr, pprior.nbr, 2 * (size_t)np, &nbr)); TRY(fit(next.O, pprior.O, 72 * (size_t)np));
      TRY(fit(next.ptr, pprior.ptr, (size_t)nc + 1, &ptr)); TRY(fit(next.ov, pprior.ov, 9 * (size_t)nc));
      TRY(fit(diag.H, cprior.H, (size_t)81 * nc)); TRY(fit(diag.g, cprior.g, (size_t)9 * nc));
      CU(cudaStreamSynchronize(stream));
      pprior.adopt(next); cprior.adopt(diag);
    }
    pprior.n = np;
    pprior.item_of = std::move(item_of);
    pprior.loss.on = false;
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
    std::vector<int> slot(L.sorted_lm.size(), -1), of_lm((size_t)L.nl_local, -1), lm, item_of((size_t)std::max(num, 0), -1);
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
      if (l < L.lm_begin || l >= L.lm_end) item_of[p] = -2;
      if (!nonzero || l < L.lm_begin || l >= L.lm_end) continue;
      const int q = (int)lm.size();
      item_of[p] = q;
      lm.push_back(l - L.lm_begin);
      slot[L.sorted_of_lm[l - L.lm_begin]] = q;
      of_lm[l - L.lm_begin] = q;
      mean.insert(mean.end(), m + 3 * (size_t)p, m + 3 * (size_t)(p + 1));
      Lsq.insert(Lsq.end(), Ls + 9 * (size_t)p, Ls + 9 * (size_t)(p + 1));
    }
    const int np = (int)lm.size();
    if (np > 0) {
      LandmarkPriorTerm next;
      TRY(fit(next.lm, lprior.lm, (size_t)np, &lm)); TRY(fit(next.mean, lprior.mean, 3 * (size_t)np, &mean));
      TRY(fit(next.L, lprior.L, 9 * (size_t)np, &Lsq)); TRY(fit(next.Lg, lprior.Lg, 12 * (size_t)np));
      TRY(fit(next.slot, lprior.slot, slot.size(), &slot)); TRY(fit(next.of_lm, lprior.of_lm, of_lm.size(), &of_lm));
      CU(cudaStreamSynchronize(stream));
      lprior.adopt(next);
    }
    lprior.n = np;
    lprior.item_of = std::move(item_of);
    lprior.loss.on = false;
    return priors_changed();
  }

  // A square-root information W (row-major 2x2) per observation of the full problem (DESIGN.md section 19).  Part of the
  // linearisation like the priors.  Every rank receives the full array and keeps the entries of its own landmark shard, in
  // slot order.  NULL, or an identity bit for bit on every observation of the shard, = the unmodified kernels
  // (D.obs_W == nullptr).  Every check runs before anything changes, so a rejected call leaves the previous information.
  int set_observation_info(const void* sqrt_info_v) override {
    const S* W = (const S*)sqrt_info_v;
    bool any = false;
    std::vector<S> w;
    if (W) {
      for (long long k = 0; k < 4 * nobs_total; ++k)
        if (!std::isfinite((double)W[k])) {
          g_err = "rba_set_observation_info: observation " + std::to_string(k / 4) + " has a non-finite sqrt_info";
          return RBA_ERR_INVALID_ARGUMENT;
        }
      static const S eye[4] = {S(1), S(0), S(0), S(1)};
      w.assign((size_t)4 * L.nslots, S(0));
      for (int s = 0; s < L.nslots; ++s) {
        if (L.slot_obs[s] < 0) continue;
        const S* src = W + 4 * (size_t)L.slot_obs[s];
        std::copy(src, src + 4, w.begin() + 4 * (size_t)s);
        any = any || std::memcmp(src, eye, sizeof(eye)) != 0;
      }
    }
    if (any) {
      DeviceBuffer<S> next; TRY(fit(next, obs.W, w.size(), &w));
      CU(cudaStreamSynchronize(stream));
      obs.W.take(next);
    }
    obs.on = any;
    su_valid = s_valid = false;  // the assembled matrix belongs to the previous rows
    return priors_changed();
  }
  // Scalars of the loss records of nslots slots (D.obs_loss): float {scale, uint32 kind} per slot; double the scales, then
  // one uint8 kind per slot, rounded up to whole doubles
  static size_t loss_records(int nslots) { return sizeof(S) == 4 ? 2 * (size_t)nslots : (size_t)nslots + ((size_t)nslots + 7) / 8; }
  // record s of the nslots records in rec (loss_records layout); NONE ignores its scale
  static void put_loss(std::vector<S>& rec, int nslots, size_t s, uint8_t k, S a) {
    const S sc = k == RBA_LOSS_NONE ? S(0) : a;
    if constexpr (sizeof(S) == 4) {
      const uint32_t k32 = k;
      rec[2 * s] = sc;
      std::memcpy(&rec[2 * s + 1], &k32, 4);
    } else {
      rec[s] = sc;
      reinterpret_cast<uint8_t*>(rec.data() + nslots)[s] = k;
    }
  }
  // The checks of rba_set_observation_loss and rba_set_prior_loss on one entry: why it is rejected ("" = accepted)
  static std::string check_loss(uint8_t kind, S a) {
    if (kind > RBA_LOSS_TUKEY) return "has kind " + std::to_string(kind) + " (must be 0..4)";
    if (kind != RBA_LOSS_NONE && !(std::isfinite((double)a) && a > S(0)))
      return "has the scale " + std::to_string((double)a) + " (must be finite and > 0)";
    return "";
  }
  // A robust loss (RBA_LOSS_*, scale) per observation of the full problem (DESIGN.md section 21).  Part of the linearisation
  // like the observation information, and landmark-owned like it: every rank receives the full arrays and keeps its own
  // shard's slots.  NULL, or the handle's own choice (robust_norm, huber_parameter) on every observation of the shard, = the
  // unmodified kernels (D.obs_loss == nullptr).  Every check runs before anything changes, so a rejected call leaves the
  // previous losses.
  int set_observation_loss(const uint8_t* kind, const void* scale_v) override {
    auto bad = [&](const std::string& what) { g_err = "rba_set_observation_loss: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (!kind != !scale_v) return bad("kind and scale must both be given or both be NULL");
    const S* a = (const S*)scale_v;
    bool any = false;
    std::vector<S> rec;
    if (kind) {
      for (long long o = 0; o < nobs_total; ++o) {
        const std::string why = check_loss(kind[o], a[o]);
        if (!why.empty()) return bad("observation " + std::to_string(o) + " " + why);
      }
      const uint8_t own = opt.robust_norm == 1 ? RBA_LOSS_HUBER : RBA_LOSS_NONE;
      const S own_a = (S)opt.huber_parameter;
      rec.assign(loss_records(L.nslots), S(0));  // padding slots: NONE
      for (int s = 0; s < L.nslots; ++s) {
        const long long o = L.slot_obs[s];
        if (o < 0) continue;
        const uint8_t k = kind[o];
        any = any || k != own || (k == RBA_LOSS_HUBER && a[o] != own_a);
        put_loss(rec, L.nslots, (size_t)s, k, a[o]);
      }
    }
    if (any) {
      DeviceBuffer<S> next; TRY(fit(next, obs.loss, rec.size(), &rec));
      CU(cudaStreamSynchronize(stream));
      obs.loss.take(next);
    }
    obs.loss_on = any;
    su_valid = s_valid = false;  // the assembled matrix belongs to the previous rows
    return priors_changed();
  }
  // One prior kind's term as rba_set_prior_loss and rba_get_prior_residuals see it: its loss, its n items, the entries of a
  // row of L (nr) and the caller's entries (num) with their items (item(p): >= 0 the item, -1 dropped, -2 other shard)
  struct PriorKindView {
    PriorLoss* loss;
    int n, nr, num;
    const std::vector<int>* item_of;  // nullptr = the cameras: item p = camera p while there are camera priors
    int item(int p, bool on) const { return item_of ? (*item_of)[p] : on ? p : -1; }
  };
  PriorKindView prior_kind_view(int32_t k) {
    if (k == RBA_PRIOR_CAMERA) return {&cprior.loss, cprior.on ? nc : 0, 9, nc, nullptr};
    if (k == RBA_PRIOR_PAIR) return {&pprior.loss, pprior.n, 6, (int)pprior.item_of.size(), &pprior.item_of};
    return {&lprior.loss, lprior.n, 3, (int)lprior.item_of.size(), &lprior.item_of};
  }
  // A robust loss per prior of one kind, in the caller's order of its setter (DESIGN.md section 22).  Part of the
  // linearisation like the priors.  NULL, or NONE on every prior, = the unmodified kernels.  Every check runs before anything
  // changes, so a rejected call leaves the previous losses.
  int set_prior_loss(int32_t which, int32_t num, const uint8_t* kind, const void* scale_v) override {
    auto bad = [&](const std::string& what) { g_err = "rba_set_prior_loss: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (which != RBA_PRIOR_CAMERA && which != RBA_PRIOR_PAIR && which != RBA_PRIOR_LANDMARK)
      return bad("prior_kind must be RBA_PRIOR_CAMERA, RBA_PRIOR_PAIR or RBA_PRIOR_LANDMARK, got " + std::to_string(which));
    const PriorKindView v = prior_kind_view(which);
    if (num != v.num)
      return bad("num is " + std::to_string(num) + ", but this prior kind has " + std::to_string(v.num) +
                 (which == RBA_PRIOR_CAMERA ? " cameras" : " entries in the last call of its setter"));
    if (!kind != !scale_v) return bad("kind and scale must both be given or both be NULL");
    const S* a = (const S*)scale_v;
    bool any = false;
    std::vector<S> rec(loss_records(v.n), S(0));
    if (kind) {
      for (int p = 0; p < num; ++p) {
        const std::string why = check_loss(kind[p], a[p]);
        if (!why.empty()) return bad("prior " + std::to_string(p) + " " + why);
      }
      for (int p = 0; p < num; ++p) {
        const int q = v.item(p, true);
        if (q < 0 || q >= v.n) continue;
        put_loss(rec, v.n, (size_t)q, kind[p], a[p]);
        any = any || kind[p] != RBA_LOSS_NONE;
      }
    }
    if (any) {
      DeviceBuffer<S> next_rec, next_Lw;
      TRY(fit(next_rec, v.loss->rec, rec.size(), &rec)); TRY(fit(next_Lw, v.loss->Lw, (size_t)v.nr * v.nr * v.n));
      CU(cudaStreamSynchronize(stream));
      v.loss->rec.take(next_rec); v.loss->Lw.take(next_Lw);
    }
    v.loss->on = any;
    return priors_changed();
  }
  // Per prior of one kind at the current state, in the caller's order (DESIGN.md section 22): L e and w.  Nothing of the
  // handle changes: the scratch is allocated for the call and freed before it returns.
  int get_prior_residuals(int32_t which, void* residual, void* robust_weight) override {
    auto bad = [&](const std::string& what) { g_err = "rba_get_prior_residuals: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (which != RBA_PRIOR_CAMERA && which != RBA_PRIOR_PAIR && which != RBA_PRIOR_LANDMARK)
      return bad("prior_kind must be RBA_PRIOR_CAMERA, RBA_PRIOR_PAIR or RBA_PRIOR_LANDMARK, got " + std::to_string(which));
    if (!residual && !robust_weight) return bad("residual and robust_weight are both NULL");
    const PriorKindView v = prior_kind_view(which);
    const size_t n = (size_t)v.n;
    std::vector<S> res(v.nr * n), w(n);
    if (n > 0) {
      DeviceBuffer<S> scratch;  // per-call
      TRY(alloc(scratch, (v.nr + 1) * n, false, false));
      S* d_res = scratch.get(); S* d_w = d_res + v.nr * n;
      const S* loss = v.loss->on ? v.loss->rec.get() : nullptr;
      const unsigned grid = (unsigned)((n + 127) / 128);
      if (which == RBA_PRIOR_CAMERA) k_prior_residuals<<<grid, 128, 0, stream>>>(camera_prior(), loss, v.n, d_res, d_w);
      else if (which == RBA_PRIOR_PAIR) k_prior_residuals<<<grid, 128, 0, stream>>>(pair_prior(), loss, v.n, d_res, d_w);
      else k_prior_residuals<<<grid, 128, 0, stream>>>(landmark_prior(), loss, v.n, d_res, d_w);
      CU(cudaMemcpyAsync(res.data(), d_res, v.nr * n * sizeof(S), cudaMemcpyDeviceToHost, stream));
      CU(cudaMemcpyAsync(w.data(), d_w, n * sizeof(S), cudaMemcpyDeviceToHost, stream));
      CU(cudaStreamSynchronize(stream));
      CU(cudaGetLastError());
    }
    for (int p = 0; p < v.num; ++p) {
      const int q = v.item(p, v.n > 0);
      if (q == -2) continue;  // a landmark prior of another shard
      for (int i = 0; i < v.nr; ++i) if (residual) ((S*)residual)[(size_t)v.nr * p + i] = q < 0 ? S(0) : res[(size_t)v.nr * q + i];
      if (robust_weight) ((S*)robust_weight)[p] = q < 0 ? S(1) : w[q];
    }
    return RBA_OK;
  }
  // Per observation at the current state, in problem order (DESIGN.md section 19).  Nothing of the handle changes: the
  // slot-ordered scratch is allocated for the call and freed before it returns.
  int get_observation_residuals(void* residual, void* robust_weight, uint8_t* flags) override {
    if (!residual && !robust_weight && !flags) {
      g_err = "rba_get_observation_residuals: residual, robust_weight and flags are all NULL";
      return RBA_ERR_INVALID_ARGUMENT;
    }
    const size_t ns = (size_t)L.nslots;
    DeviceBuffer<char> scratch;  // per-call
    TRY(alloc(scratch, ns * (3 * sizeof(S) + 1), false, false));
    S* d_res = (S*)scratch.get(); S* d_hw = d_res + 2 * ns; uint8_t* d_fl = (uint8_t*)(d_hw + ns);
    k_obs_residuals<S><<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(D, ko, d_res, d_hw, d_fl);
    std::vector<S> res(2 * ns), hw(ns);
    std::vector<uint8_t> fl(ns);
    CU(cudaMemcpyAsync(res.data(), d_res, 2 * ns * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(hw.data(), d_hw, ns * sizeof(S), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(fl.data(), d_fl, ns, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    CU(cudaGetLastError());
    for (size_t s = 0; s < ns; ++s) {
      const long long ob = L.slot_obs[s];
      if (ob < 0) continue;
      if (residual) { ((S*)residual)[2 * ob] = res[2 * s]; ((S*)residual)[2 * ob + 1] = res[2 * s + 1]; }
      if (robust_weight) ((S*)robust_weight)[ob] = hw[s];
      if (flags) flags[ob] = fl[s];
    }
    return RBA_OK;
  }

  // Triangulation of the listed landmarks from the current cameras (DESIGN.md section 25): one k_triangulate launch over the
  // entries of this shard, in the length-sorted order.  Every check runs before any device work.  A state change: the error
  // cache, the linearisation and the device-resident increment are discarded; the backup is not touched.
  int triangulate(const rba_triangulate_opts* o, int32_t num, const int32_t* lm_idx, uint8_t* status, double* angle,
                  double* cost) override {
    auto bad = [&](const std::string& what) { g_err = "rba_triangulate_landmarks: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (!o) return bad("o is NULL");
    if (o->mode < 1 || o->mode > 3) return bad("mode must be 1..3 (RBA_TRIANGULATE_* bits), got " + std::to_string(o->mode));
    if (o->max_iterations < 0) return bad("max_iterations must be >= 0, got " + std::to_string(o->max_iterations));
    if (!std::isfinite(o->min_angle) || o->min_angle < 0) return bad("min_angle must be finite and >= 0");
    if (!std::isfinite(o->function_tolerance) || o->function_tolerance < 0) return bad("function_tolerance must be finite and >= 0");
    if (num < 0) return bad("num must be >= 0, got " + std::to_string(num));
    if (!lm_idx && num != nl_total)
      return bad("lm_idx is NULL, so num must be the number of landmarks " + std::to_string(nl_total) + ", got " + std::to_string(num));
    std::vector<uint8_t> seen(lm_idx ? (size_t)nl_total : 0, 0);
    std::vector<std::pair<int, int>> mine;  // (sorted index, caller position) of this shard's entries
    for (int p = 0; p < num; ++p) {
      const int l = lm_idx ? lm_idx[p] : p;
      if (lm_idx) {
        if (l < 0 || l >= nl_total) return bad("entry " + std::to_string(p) + " has a landmark index outside [0, " + std::to_string(nl_total) + ")");
        if (seen[l]) return bad("entry " + std::to_string(p) + " repeats landmark " + std::to_string(l));
        seen[l] = 1;
      }
      if (l >= L.lm_begin && l < L.lm_end) mine.push_back({L.sorted_of_lm[l - L.lm_begin], p});
    }
    std::sort(mine.begin(), mine.end());
    const size_t ni = mine.size();
    if (ni > 0) {
      std::vector<TriItem> items(ni);
      for (size_t k = 0; k < ni; ++k) {
        const int sidx = mine[k].first;
        const TileInfo& T = L.tiles[L.tile_of_sorted[sidx]];
        items[k] = {L.sorted_lm[sidx], sidx, T.slot_base + (sidx - T.lm_base) * T.n, T.n};
      }
      DeviceBuffer<char> scratch;  // per-call: the rays, the items, the outputs and the validity bytes
      const size_t ray_b = (size_t)L.nslots * sizeof(double4), item_b = ni * sizeof(TriItem);
      TRY(alloc(scratch, ray_b + item_b + ni * (2 * sizeof(double) + 1) + (size_t)L.nslots, false, false));
      double4* d_ray = (double4*)scratch.get();
      TriItem* d_items = (TriItem*)(scratch.get() + ray_b);
      double* d_angle = (double*)(scratch.get() + ray_b + item_b);
      double* d_cost = d_angle + ni;
      uint8_t* d_status = (uint8_t*)(d_cost + ni);
      uint8_t* d_vb = d_status + ni;
      CU(cudaMemcpyAsync(d_items, items.data(), item_b, cudaMemcpyHostToDevice, stream));
      const TriOpts to{o->mode, o->max_iterations, o->min_angle, o->function_tolerance};
      k_triangulate<S><<<grid_for((long long)ni, 4, 16), 128, 0, stream>>>(D, ko, to, d_items, (int)ni, d_ray, d_vb, d_status, d_angle, d_cost);
      ++launches;
      std::vector<uint8_t> st(ni);
      std::vector<double> an(ni), co(ni);
      CU(cudaMemcpyAsync(st.data(), d_status, ni, cudaMemcpyDeviceToHost, stream));
      CU(cudaMemcpyAsync(an.data(), d_angle, ni * sizeof(double), cudaMemcpyDeviceToHost, stream));
      CU(cudaMemcpyAsync(co.data(), d_cost, ni * sizeof(double), cudaMemcpyDeviceToHost, stream));
      CU(cudaStreamSynchronize(stream));
      CU(cudaGetLastError());
      for (size_t k = 0; k < ni; ++k) {
        const int p = mine[k].second;
        if (status) status[p] = st[k];
        if (angle) angle[p] = an[k];
        if (cost) cost[p] = co[k];
      }
    }
    ++state_version;
    linearized = false;
    damping_valid = false;
    have_inc = false;
    error_cache_valid = false;
    return RBA_OK;
  }

  // Resection of the listed cameras' units from the current landmarks (DESIGN.md section 26): one k_resect launch, a CTA
  // per unit, the units in decreasing observation count.  Every check runs before any device work.  A state change like
  // triangulate: the error cache, the linearisation and the device-resident increment are discarded; the backup is not
  // touched.
  int resect(const rba_resect_opts* o, int32_t num, const int32_t* cam_idx, uint8_t* status, int32_t* points,
             double* cost) override {
    auto bad = [&](const std::string& what) { g_err = "rba_resect_cameras: " + what; return RBA_ERR_INVALID_ARGUMENT; };
    if (!o) return bad("o is NULL");
    const int md = o->mode;
    if ((md & ~7) || !(md & 3) || ((md & RBA_RESECT_INTRINSICS) && !(md & RBA_RESECT_REFINE)))
      return bad("mode must be LINEAR and / or REFINE, INTRINSICS only with REFINE (RBA_RESECT_* bits), got " + std::to_string(md));
    if (o->max_iterations < 0) return bad("max_iterations must be >= 0, got " + std::to_string(o->max_iterations));
    if (!std::isfinite(o->function_tolerance) || o->function_tolerance < 0) return bad("function_tolerance must be finite and >= 0");
    if (num < 0) return bad("num must be >= 0, got " + std::to_string(num));
    if (!cam_idx && num != nc)
      return bad("cam_idx is NULL, so num must be the number of cameras " + std::to_string(nc) + ", got " + std::to_string(num));
    std::vector<uint8_t> seen(cam_idx ? (size_t)nc : 0, 0);
    for (int p = 0; p < num && cam_idx; ++p) {
      const int c = cam_idx[p];
      if (c < 0 || c >= nc) return bad("entry " + std::to_string(p) + " has a camera index outside [0, " + std::to_string(nc) + ")");
      if (seen[c]) return bad("entry " + std::to_string(p) + " repeats camera " + std::to_string(c));
      seen[c] = 1;
    }
    if (opt.nranks > 1) {
      g_err = "rba_resect_cameras: a sharded handle is not supported (a camera's observations span every shard)";
      return RBA_ERR_UNSUPPORTED;
    }
    // the units: a rig of >= 2 cameras is one unit led by its lead, its members ascending; any other camera is its own
    auto lead_of = [&](int c) { return rig.n && rig.host_lead[c] >= 0 ? rig.host_lead[c] : c; };
    std::vector<int> unit_of((size_t)nc, -1), unit_lead, caller_unit((size_t)num);
    for (int p = 0; p < num; ++p) {
      const int ld = lead_of(cam_idx ? cam_idx[p] : p);
      if (unit_of[ld] < 0) { unit_of[ld] = (int)unit_lead.size(); unit_lead.push_back(ld); }
      caller_unit[p] = unit_of[ld];
    }
    const size_t nu = unit_lead.size();
    std::vector<std::vector<int>> members(nu);
    for (int c = 0; c < nc; ++c)
      if (unit_of[lead_of(c)] >= 0) members[unit_of[lead_of(c)]].push_back(c);
    const auto& cp = L.csr_obs.cam_ptr;
    std::vector<long long> nobs(nu, 0);
    for (size_t u = 0; u < nu; ++u)
      for (int c : members[u]) nobs[u] += cp[c + 1] - cp[c];
    std::vector<int> order(nu);
    for (size_t u = 0; u < nu; ++u) order[u] = (int)u;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return nobs[a] != nobs[b] ? nobs[a] > nobs[b] : unit_lead[a] < unit_lead[b]; });
    std::vector<int> pos_of(nu);
    std::vector<ResItem> items(nu);
    std::vector<ResMember> mem;
    for (size_t k = 0; k < nu; ++k) {
      const int u = order[k], ld = unit_lead[u];
      pos_of[u] = (int)k;
      const unsigned fl = held.host.empty() ? 0u : held.host[ld];
      unsigned fr = (fl & RBA_FIX_POSE) ? 0u : 0x3fu;
      const bool single = members[u].size() == 1, grouped = grp.n && grp.host_lead[ld] >= 0;
      if ((md & RBA_RESECT_INTRINSICS) && single && !grouped) fr |= ~fixed_entry_mask(fl | RBA_FIX_POSE) & 0x1c0u;
      items[k] = {(int)mem.size(), (int)members[u].size(), ld, fr};
      for (int c : members[u]) mem.push_back({c, cp[c], cp[c + 1]});
    }
    if (nu > 0) {
      DeviceBuffer<char> scratch;  // per-call: the snapshot, the items, the members, their M_j and A_j, the outputs, the validity bytes
      const size_t snap_b = (size_t)10 * nc * sizeof(S), item_b = nu * sizeof(ResItem), mem_b = mem.size() * sizeof(ResMember);
      const size_t mx_b = mem.size() * RES_MX * sizeof(double), out_b = nu * (sizeof(double) + sizeof(int) + 1);
      auto up8 = [](size_t b) { return (b + 15) & ~(size_t)15; };
      TRY(alloc(scratch, up8(snap_b) + up8(item_b) + up8(mem_b) + up8(mx_b) + up8(out_b) + (size_t)L.nslots, false, false));
      char* at = scratch.get();
      S* d_snap = (S*)at; at += up8(snap_b);
      ResItem* d_items = (ResItem*)at; at += up8(item_b);
      ResMember* d_mem = (ResMember*)at; at += up8(mem_b);
      double* d_mx = (double*)at; at += up8(mx_b);
      double* d_cost = (double*)at;
      int* d_points = (int*)(d_cost + nu);
      uint8_t* d_status = (uint8_t*)(d_points + nu);
      uint8_t* d_vb = (uint8_t*)(at + up8(out_b));
      CU(cudaMemcpyAsync(d_snap, D.cams, snap_b, cudaMemcpyDeviceToDevice, stream));
      CU(cudaMemcpyAsync(d_items, items.data(), item_b, cudaMemcpyHostToDevice, stream));
      CU(cudaMemcpyAsync(d_mem, mem.data(), mem_b, cudaMemcpyHostToDevice, stream));
      ResTerms<S> T{};
      T.snap = d_snap;
      T.slots = d_csr_obs_slots;
      if (rig.n) T.R = rigs();
      if (sen.n) T.Z = sensors();
      if (cprior.on) { T.cp_mean = cprior.mean.get(); T.cp_L = cprior.L.get(); T.cp_loss = cprior.loss.on ? cprior.loss.rec.get() : nullptr; }
      if (pprior.n > 0) {
        T.pp_ij = pprior.ij.get(); T.pp_mean = pprior.mean.get(); T.pp_L = pprior.L.get();
        T.pp_loss = pprior.loss.on ? pprior.loss.rec.get() : nullptr; T.pp_ptr = pprior.ptr.get(); T.pp_item = pprior.item.get();
        T.pp_n = pprior.n;
      }
      const ResOpts ro{md, o->max_iterations, o->function_tolerance};
      k_resect<S><<<(unsigned)nu, RES_THREADS, 0, stream>>>(D, ko, ro, T, d_items, d_mem, d_mx, d_vb, d_status, d_points, d_cost);
      ++launches;
      std::vector<uint8_t> st(nu);
      std::vector<int> pt(nu);
      std::vector<double> co(nu);
      CU(cudaMemcpyAsync(st.data(), d_status, nu, cudaMemcpyDeviceToHost, stream));
      CU(cudaMemcpyAsync(pt.data(), d_points, nu * sizeof(int), cudaMemcpyDeviceToHost, stream));
      CU(cudaMemcpyAsync(co.data(), d_cost, nu * sizeof(double), cudaMemcpyDeviceToHost, stream));
      CU(cudaStreamSynchronize(stream));
      CU(cudaGetLastError());
      for (int p = 0; p < num; ++p) {
        const int k = pos_of[caller_unit[p]];
        if (status) status[p] = st[k];
        if (points) points[p] = pt[k];
        if (cost) cost[p] = co[k];
      }
    }
    ++state_version;
    linearized = false;
    damping_valid = false;
    have_inc = false;
    error_cache_valid = false;
    return RBA_OK;
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
    auto ke = k_error_instance(D.obs_W, D.obs_loss);  // OBSW: the whitened residuals (section 19); OBSL: their own losses (section 21)
    ke<<<EBLOCKS, 256, 0, stream>>>(D, ko, d_epart, d_flags);
    k_sum_partials<6><<<1, 256, 0, stream>>>(d_epart, EBLOCKS, d_red);
    launches += 2;
    // (each prior's cost is rho(|L e|^2)/2 of its loss while its kind has losses, DESIGN.md section 22)
    if (lprior.n > 0) {  // + this shard's landmark priors' 1/2 |L e|^2, BEFORE the sum over the shards (landmark-owned)
      rc = prior_cost(landmark_prior(), lprior.n, lprior.loss); if (rc) return rc;
    }
    rc = allreduce_scalars(6); if (rc) return rc;
    if (cprior.on) {  // + sum of 1/2 |L e|^2, once, after the sum over the shards
      rc = prior_cost(camera_prior(), nc, cprior.loss); if (rc) return rc;
    }
    if (pprior.n > 0) {  // + the pair priors' 1/2 |L e|^2, likewise
      rc = prior_cost(pair_prior(), pprior.n, pprior.loss); if (rc) return rc;
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
    const int n_pairs = pprior.n, n_groups = grp.n;
    int rc = start(ev_stage1); if (rc) return rc;
    CU(cudaMemsetAsync(d_flags, 0, 4 * sizeof(int), stream));
    // pass A: squared column norms of the weighted pose Jacobians -> pose_jacobian_scaling_
    auto kn = k_jp_norms_instance(D.obs_W, D.obs_loss);
    kn<<<grid_for(L.nslots, 256, 8), 256, 0, stream>>>(D, ko, d_flags);
    ++launches;
    rc = camera_reduce(d_csr_obs_slots, d_csr_obs_items, n_obs_items, d_csr_obs_item_ptr, D.diag2); if (rc) return rc;
    // (the priors' losses: sqrt(w) L in place of L, DESIGN.md section 22)
    if (cprior.on) {  // prior Jacobian and its column norms (scaling from the whole Jacobian), after the sum over the shards
      const S* Lc = weighted_L(camera_prior(), nc, cprior.loss);
      k_prior_linearize<S><<<(nc + 127) / 128, 128, 0, stream>>>(D.cams, cprior.mean.get(), Lc, nc, D.diag2, cprior.A.get(), cprior.r.get());
      ++launches;
    }
    if (n_pairs > 0) {  // pair-prior blocks and their column norms, likewise
      const S* Lp = weighted_L(pair_prior(), n_pairs, pprior.loss);
      k_pair_linearize<S><<<(n_pairs + 127) / 128, 128, 0, stream>>>(D.cams, pprior.ij.get(), pprior.mean.get(), Lp, n_pairs, pprior.A.get(), pprior.r.get());
      k_pair_diag2<S><<<(nc + 127) / 128, 128, 0, stream>>>(pprior.A.get(), pprior.ptr.get(), pprior.item.get(), nc, D.diag2);
      launches += 2;
    }
    if (n_groups) {  // the merged intrinsics columns' norms for every member, after the sum over the shards and the priors
      k_group_sum_diag2<S><<<n_groups, GROUP_THREADS, 0, stream>>>(D.diag2, groups());
      ++launches;
    }
    k_scaling<S><<<(9 * nc + 255) / 256, 256, 0, stream>>>(D.diag2, D.scaling, 9 * nc, (S)ko.jacobi_eps);
    // pass B: linearize (scaled) + Jl scaling + Householder QR + panel write
    // (+ the landmark priors' column norms, L~ and g: the LMP instances; + the observation information: the OBSW instances;
    // + the observation losses: the OBSL instances).  ref: ipp:149-163 selects perform_qr_givens
    auto k1 = k1_instance(!opt.use_householder_marginalization, D.lmp_slot, D.obs_W, D.obs_loss);
    if (lprior.n > 0) weighted_L(landmark_prior(), lprior.n, lprior.loss);  // into D.lmp_L while the losses are on
    k1<<<tile_grid(k1_max_blocks), TILE_WARPS * 32, k1_smem, stream>>>(D, ko, k1_sc, d_flags, order_k1);
    launches += 2;
    if (opt.preconditioner_type == 0 || opt.solver_type == 2) {
      // JACOBI: D (sum Jp^T Jp) D from the stored scaled Jacobians (Power-SC: these blocks are Hpp, sc/linearization_power_sc.hpp:92-128) (ref: ipp:554-569, block_sparse_matrix.hpp:89-100)
      rc = precond_blocks(0, D.jblocks, nullptr, true); if (rc) return rc;
    }
    const bool jac = opt.preconditioner_type == 0 || opt.solver_type == 2;
    if (cprior.on) {  // scaled prior Jacobian, A^T A (+ into the JACOBI blocks), A^T r
      k_prior_scale<S><<<(nc + 127) / 128, 128, 0, stream>>>(cprior.A.get(), cprior.r.get(), D.scaling, nc, cprior.H.get(), cprior.g.get(), jac ? D.jblocks : nullptr);
      ++launches;
    }
    if (n_pairs > 0) {  // scaled pair blocks; their diagonal blocks and A^T r added to the absolute priors', the O_ij of every edge
      k_pair_scale<S><<<(n_pairs + 127) / 128, 128, 0, stream>>>(pprior.A.get(), pprior.ij.get(), D.scaling, n_pairs);
      k_pair_accum<S><<<(nc + 127) / 128, 128, 0, stream>>>(pprior.A.get(), pprior.r.get(), pprior.ptr.get(), pprior.item.get(), nc, (int)cprior.on,
                                                            cprior.H.get(), cprior.g.get(), jac ? D.jblocks : nullptr, pprior.O.get());
      launches += 2;
    }
    if (rig.n) {
      // (rigs: D_u from the per-camera Gram of the scaled rows and P~ of every member, DESIGN.md section 23.  The JACOBI blocks
      // hold the observation Gram and the priors' H; with SCHUR_JACOBI they are unused, so they take the observation Gram
      // here and the priors' H is added in k_rig_scaling)
      if (!jac) { rc = precond_blocks(0, D.jblocks, nullptr, true); if (rc) return rc; }
      // (sensors, section 24: A_j of their cameras from the state first, then D_s and Q~ in the blocks after the rigs')
      if (sen.n) TRY(sensor_tie());
      const S* pH = jac ? nullptr : (const S*)D.prior_H;
      if (sen.n)
        k_rig_scaling<S, true><<<rig.n + sen.n, GROUP_THREADS, 0, stream>>>(D.jblocks, pH, D, rigs(), (S)ko.jacobi_eps, sensors());
      else
        k_rig_scaling<S><<<rig.n, GROUP_THREADS, 0, stream>>>(D.jblocks, pH, D, rigs(), (S)ko.jacobi_eps, NoSensors{});
      ++launches;
    }
    if (panel_form()) {
      // rows 3..2n-1 of the Q2 panels do not change with lambda: their part of the gradient (ipp:443-466) and of the
      // SCHUR_JACOBI blocks (ipp:520-552) is accumulated once per linearisation (this shard only; the sum over the
      // shards happens in solve() together with the damping-row part)
      const int want_blocks = opt.preconditioner_type >= 1 ? 1 : 0;
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

  // How the operator's output reaches the vector step, decided in one place (handover()):
  enum class Handover {
    Assembled,  // S is assembled for this solve's lambda (setup_assembled): k_rcs_spmv writes D.y
    Partials,   // one GPU, PCG, while a cluster CTA's share of the cameras fits the vector kernel's registers (9 ceil(nc /
                // cluster) <= VEC_THREADS VEC_EPT: <= 1808 cameras with 16 CTAs, <= 904 with 8): k_cam_reduce writes the
                // per-segment sums and k_pcg_vec adds them in the order of k_cam_reduce_final's last arriver (bit-identical,
                // without its arrival counters and fences)
    Counter,    // one GPU otherwise (the power series, and larger camera counts such as Final-13682, the combination
                // measured there): k_cam_reduce_final<false> writes D.y
    Peer,       // several ranks, peers mapped (rba_ipc_import): k_cam_reduce_final<true> into every rank's staging area,
                // which k_pcg_vec sums
    Nccl,       // several ranks otherwise: D.y cleared, k_cam_reduce_final<false>, all-reduced, vector step without PDL
  };
  // k_cam_reduce_final never writes a camera without observations in this shard.  So Counter needs D.y cleared once per
  // solve and before rba_right_multiply (an earlier call may have left other values: rba_right_multiply stores lambda x
  // there), and Nccl before every application (the in-place all-reduce would carry the previous sum into the next).  The
  // others need no clear: k_rcs_spmv writes every camera, k_pcg_vec takes 0 for a camera without segments, and a peer
  // staging slot that is never written stays zero.
  // With intrinsics groups or rigs the operator output is contracted (k_group_contract, k_rig_contract) between the
  // reduction and the vector step, so it must exist as one vector: Partials and Peer, which sum the segments inside
  // k_pcg_vec, give way to Counter / Nccl.
  Handover handover() const {
    if (s_valid) return Handover::Assembled;
    if (grp.n || rig.n) return opt.nranks > 1 ? Handover::Nccl : Handover::Counter;
    if (opt.nranks > 1) return peer_ok ? Handover::Peer : Handover::Nccl;
    const bool vec_cached = 9 * ((nc + pcg_cluster - 1) / pcg_cluster) <= VEC_THREADS * VEC_EPT;
    return pcg_partials && vec_cached && opt.solver_type != 2 ? Handover::Partials : Handover::Counter;
  }
  // One operator application H x (e0_only: the implicit operator's E_0 x alone) and the reduction of hand-over h; the caller
  // then launches its vector kernel.  In a solve the kernels return at once when it has ended, and those that may are
  // launched dependent on their predecessor.
  int apply_operator(const S* xvec, Handover h, bool in_solve, int e0_only = 0) {
    const int* done = in_solve ? &d_state->done : nullptr;
    const bool pdl = in_solve;
    ++tm.matvec_launches;
    if (h == Handover::Assembled) {
      const bool p = pdl && !s_fresh;
      s_fresh = false;
      return launch_ex(k_rcs_spmv<S>, spmv_grid, SPMV_CLASSES * 32, 0, p, 1, (const SpmvChunk*)d_spmv_chunks, (const int*)d_spmv_chunk_ptr,
                       (const int*)d_asm_col, (const S*)d_asm_S, xvec, D.y, done, (int)p);
    }
    if (panels) {  // yobs = P^T P x
      if (L.n_items_large > 0) {
        k_matvec_large<S, K4_WARPS, KPMAX><<<grid_for(L.n_items_large, K4_WARPS, 4), K4_WARPS * 32, k4_smem_small, stream>>>(
            D, d_items, 0, L.n_items_large, L.k4_scratch_per_warp, xvec, done);
        ++launches;
      }
      const bool p = pdl && L.n_items_large == 0;
      if (n_dealt > L.n_items_large)
        TRY(launch_ex(k_matvec_small_tma<S, K4_WARPS, K4_NS, K4_STAGE>, tma_grid, K4_WARPS * 32, K4_SMEM_TMA, p, 1, D, (const MatvecItem*)d_items, L.n_items_large, n_dealt, xvec, done, (int)p));
    } else {
      const int ntl = (int)L.tiles.size();
      const bool p = pdl && imp_tile_split == ntl;  // a single kernel between the PCG vector step and the reduction
      if (imp_tile_split > 0)
        TRY(launch_ex((k_matvec_implicit_tma<S, IMP_WARPS, IMP_MAXSLOTS, IMP_NS>), imp_grid, IMP_WARPS * 32, imp_smem, p, 1, D, imp_tile_split, xvec, done, (int)p, e0_only));
      if (imp_tile_split < ntl)
        TRY(launch_ex(k_matvec_implicit<S>, (ntl - imp_tile_split + TILE_WARPS - 1) / TILE_WARPS, TILE_WARPS * 32, 0, false, 1, D, imp_tile_split, xvec, done, 0, e0_only));
    }
    const int grid = grid_for(n_op_items, 8, 8);
    if (h == Handover::Partials)
      return launch_ex(k_cam_reduce<S>, grid, 256, 0, pdl, 1, (const S*)D.yobs, op_slots, op_items, n_op_items, D.partial, done, (int)pdl);
    if (h == Handover::Peer) ++ar_seq;
    if (h == Handover::Nccl) CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));
    auto kern = h == Handover::Peer ? k_cam_reduce_final<S, true> : k_cam_reduce_final<S, false>;
    TRY(launch_ex(kern, grid, 256, 0, pdl, 1, (const S*)D.yobs, op_slots, op_items, n_op_items, op_item_ptr, D.partial, d_cam_cnt, D.y, done, (int)pdl, pc, ar_seq, nc));
    return h == Handover::Nccl ? allreduce(D.y, (size_t)9 * nc) : RBA_OK;
  }
  // one operator application outside PCG (rba_right_multiply, rba_time_matvec): this shard's H x in D.y
  int matvec_launch(const S* xvec, bool clear_y) {
    const Handover h = handover() == Handover::Assembled ? Handover::Assembled : Handover::Counter;
    if (clear_y && h == Handover::Counter) CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));
    return apply_operator(xvec, h, false);
  }
  // the PCG vector step; pair priors: O v of the step's vector (v = x in the refresh's second half, else p) into D.pair_ov first
  int pcg_vec(int i, int mode, bool pdl, int is_last, S lambda, bool fused_ar = false, bool from_partials = false) {
    PeerComm c = pc;
    if (!fused_ar) c.nranks = 1;
    DevPtrs<S> Dv = D;
    if (grp.n || rig.n) {  // the contracted output, which holds the prior terms already (k_group_contract, k_rig_contract)
      Dv.y = tied_y(); Dv.prior_H = nullptr; Dv.pair_ov = nullptr;
    }
    if (clu.on) {  // CLUSTER_JACOBI: L^-1 S L^-T (k_cluster_fwd wrote it whole into yh), L^-1 b, the masked identity blocks
      Dv.y = clu.yh; Dv.b = clu.bh; Dv.inv = clu.eye; Dv.prior_H = nullptr; Dv.pair_ov = nullptr;
      lambda = S(0);
      from_partials = false;
    }
    if (Dv.pair_ov && mode != 3) TRY(pair_ov(mode == 2 ? D.x : D.p, pdl));
    auto kern = Dv.pair_ov ? k_pcg_vec<S, true, true> : Dv.prior_H ? k_pcg_vec<S, true> : k_pcg_vec<S, false>;
    return launch_ex(kern, pcg_cluster, VEC_THREADS, 0, pdl, pcg_cluster, Dv, d_state, lambda, i, mode, (double)opt.eta,
                     (int)opt.min_linear_solver_iterations, is_last, (int)pdl, c, ar_seq, from_partials ? op_item_ptr : (const int*)nullptr, d_prog);
  }
  // D.pair_ov = sum_j O_ij v_j (k_pair_ov), ahead of the vector step that consumes it
  int pair_ov(const S* v, bool pdl) {
    return launch_ex(k_pair_ov<S>, (9 * nc + 255) / 256, 256, 0, pdl, 1, D, (const PcgState*)d_state, v);
  }
  // one operator application inside PCG (H v for v = p in mode 0/1, x in mode 2) and the vector step after it
  // (intrinsics groups: H_u v = P^T H P v, with P v in grp.ve and P^T (H P v) in grp.y; rigs: P~^T K P~ v likewise in rig.ve
  // and rig.y; both: P~ v into rig.ve, P of it in place, the group contraction into grp.y and the rigs' in place there)
  int pcg_step(int i, int mode, int is_last, S lambda, Handover h) {
    const S* v = mode == 2 ? D.x : D.p;
    if (clu.on) {  // CLUSTER_JACOBI (DESIGN.md section 28): S applied to w = L^-T v, then L^-1 of its output
      cluster_back(v, clu.w, &d_state->done);
      TRY(apply_operator(clu.w, h, true));
      k_cluster_fwd<S><<<clu.ncl, CLUSTER_THREADS, cluster_factor_smem(clu.max_k), stream>>>(
          cluster_view(), D, D.y, h == Handover::Partials ? op_item_ptr : nullptr, clu.w, lambda, clu.yh, &d_state->done);
      ++launches;
      return pcg_vec(i, mode, true, is_last, lambda);
    }
    if (rig.n) {
      TRY(rig_expand(v, rig.ve.get(), true));
      v = rig.ve.get();
    }
    if (grp.n) {
      S* ve = rig.n ? rig.ve.get() : grp.ve.get();
      TRY(group_expand(v, ve, true));
      v = ve;
    }
    TRY(apply_operator(v, h, true));
    const bool pdl = h != Handover::Nccl;
    if (grp.n)
      TRY(launch_ex(k_group_contract<S>, (nc + GROUP_THREADS - 1) / GROUP_THREADS + grp.n, GROUP_THREADS, 0, pdl, 1,
                    D, v, grp.y.get(), groups(), (nc + GROUP_THREADS - 1) / GROUP_THREADS, (const PcgState*)d_state));
    const S* in = grp.n ? (const S*)grp.y.get() : (const S*)nullptr;
    if (rig.n && sen.n)  // (out of place, from the groups' output into rig.y)
      TRY(launch_ex(k_rig_contract<S, true>, rig_ncb() + rig.n + sen.n, GROUP_THREADS, 0, pdl, 1, D, v, in, tied_y(), rigs(), rig_ncb(),
                    (const PcgState*)d_state, sensors()));
    else if (rig.n)
      TRY(launch_ex(k_rig_contract<S>, rig_ncb() + rig.n, GROUP_THREADS, 0, pdl, 1, D, v, in, tied_y(), rigs(), rig_ncb(),
                    (const PcgState*)d_state, NoSensors{}));
    return pcg_vec(i, mode, h != Handover::Nccl, is_last, lambda, h == Handover::Peer, h == Handover::Partials);
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
  // kernels with e0_only), the per-camera reduction of hand-over h (Counter) and k_power_vec; the device convergence flag
  // is polled like in PCG.
  int power_enqueue(Handover h, void* inc_out) {
    TRY(start(ev_pcg));
    CU(cudaMemsetAsync(d_state, 0, sizeof(PcgState), stream));
    const int order = opt.power_order;
    // pair priors: the series on Hpp^-1 (E_0 - O), O p from k_pair_ov ahead of each term (DESIGN.md section 15)
    auto kern = D.pair_ov ? k_power_vec<S, true> : k_power_vec<S, false>;
    TRY(launch_ex(kern, pcg_cluster, VEC_THREADS, 0, false, pcg_cluster, D, d_state, 0, (double)opt.eta, 0, 0));
    TRY(enqueue_polled(order, opt.pcg_check_period, [&](int i) -> int {
      TRY(apply_operator(D.p, h, true, 1));
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
      auto k = panel_form() ? (lmp ? k_stage2<S, true, true> : k_stage2<S, true>) : (lmp ? k_stage2<S, false, true> : k_stage2<S, false>);
      k<<<tile_grid(k2_max_blocks), TILE_WARPS * 32, k2_smem, stream>>>(D, lambda, k2_sc, (int)panels);
    }
    ++launches;
    s_valid = su_new = false;  // S of the previous lambda; rebuilt if this solve runs long enough (solve_enqueue)
    rc = camera_reduce(d_csr_obs_slots, d_csr_obs_items, n_obs_items, d_csr_obs_item_ptr, D.b, panel_form() ? D.b0 : nullptr); if (rc) return rc;
    const bool power = opt.solver_type == 2;
    // (CLUSTER_JACOBI: the SCHUR_JACOBI blocks are its diagonal blocks)
    const bool schur = opt.preconditioner_type >= 1 && !power;  // Power-SC inverts Hpp = sum Jp^T Jp + lambda I instead
    if (schur) { rc = panel_form() ? precond_blocks(2, D.blocks, D.blocks0, true) : precond_blocks(1, D.blocks, nullptr, true); if (rc) return rc; }
    rc = stop(ev_stage2); if (rc) return rc;
    rc = start(ev_precond); if (rc) return rc;
    // pose damping lambda*I added to the blocks, then explicit inverse (ref: linearization_qr.hpp:796-802, linearizor_qr.cpp:228-237)
    // (+ the masking of the held camera parameters, D.cam_fixed; + the camera priors: A^T A into the SCHUR_JACOBI blocks -- the
    // JACOBI blocks hold it already -- and A^T r into b, both after the sum over the shards and before the masking)
    if (grp.n || rig.n) {
      // (intrinsics groups, rigs: the priors' terms, the contraction of b and the merged blocks first, into D.blocks; DESIGN.md
      // sections 18 and 23.  With both, the rigs' pass runs on the groups' output, whose priors' terms are in already)
      const int ncb = (nc + GROUP_THREADS - 1) / GROUP_THREADS, n_groups = grp.n;
      const S* src = schur ? D.blocks : D.jblocks;
      const S* pH = schur ? (const S*)D.prior_H : nullptr;
      const S* pg = D.prior_H ? (const S*)cprior.g.get() : nullptr;
      if (grp.n) {
        k_group_precond<S><<<ncb + n_groups, GROUP_THREADS, 0, stream>>>(src, pH, pg, D.b, D.blocks, groups(), nc, ncb);
        src = D.blocks; pH = nullptr; pg = nullptr;
      }
      if (rig.n && sen.n) {  // (sensors: out of place, from copies of the blocks and b)
        CU(cudaMemcpyAsync(sen.blk.get(), src, (size_t)81 * nc * sizeof(S), cudaMemcpyDeviceToDevice, stream));
        CU(cudaMemcpyAsync(sen.b.get(), D.b, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToDevice, stream));
        k_rig_precond<S, true><<<ncb + rig.n + sen.n, GROUP_THREADS, 0, stream>>>(sen.blk.get(), pH, pg, D.b, D.blocks, rigs(), nc, ncb,
                                                                                 sensors());
      } else if (rig.n) {
        k_rig_precond<S><<<ncb + rig.n, GROUP_THREADS, 0, stream>>>(src, pH, pg, D.b, D.blocks, rigs(), nc, ncb, NoSensors{});
      }
      k_precond_invert<S><<<(nc + 63) / 64, 64, 0, stream>>>(D.blocks, lambda, nc, schur ? D.blocks : nullptr, D.inv, tied_fixed(), D.b);
      launches += 1 + (grp.n > 0) + (rig.n > 0);
    } else {
      k_precond_invert<S><<<(nc + 63) / 64, 64, 0, stream>>>(schur ? D.blocks : D.jblocks, lambda, nc, schur ? D.blocks : nullptr, D.inv,
                                                             D.cam_fixed, D.b, schur ? (const S*)D.prior_H : nullptr,
                                                             D.prior_H ? (const S*)cprior.g.get() : nullptr);
      ++launches;
    }
    if (clu.on && !held.all) TRY(cluster_build());  // the cluster blocks and their factors (CLUSTER_JACOBI, section 28)
    rc = stop(ev_precond); if (rc) return rc;
    last_lambda = lambda;
    damping_valid = true;
    if (held.all) {
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
    if (opt.linear_solver_type == 1) return dense_enqueue((double)lambda, inc_out);  // DENSE_SCHUR: no PCG (section 27)
    Handover h = handover();
    if (h == Handover::Counter) CU(cudaMemsetAsync(D.y, 0, (size_t)9 * nc * sizeof(S), stream));  // see handover()
    if (power) return power_enqueue(h, inc_out);
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
      if (i % period == 0) {
        TRY(pcg_step(i, 1, 0, lambda, h));
        return pcg_step(i, 2, is_last, lambda, h);
      }
      return pcg_step(i, 0, is_last, lambda, h);
    };
    if (h == Handover::Nccl) {
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
          // the solve has run asm_switch - 1 iterations: from here on S x (S_u once per linearisation, then S for lambda).
          // The host may enqueue this after the solve has ended (one of the no-op iterations that follow the end): then
          // the assembly kernels do nothing and solve_finish withdraws what is set here.
          su_new = !su_valid;
          if (su_new) assemble(0);
          assemble(1);
          su_valid = s_valid = s_fresh = true;
          h = handover();
        }
        rc = enqueue_iteration(i); if (rc) return rc;
      }
    }
    if (clu.on) cluster_back(D.inc, D.inc, nullptr);  // inc = -L^-T x^ (CLUSTER_JACOBI)
    TRY(tie_expand(D.inc));  // inc = P u for the back-substitution, the update and inc_out
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
    if (s_valid && h_state[0].iter < asm_switch) {
      // the solve ended before iteration asm_switch, so the assembly enqueued after its end did nothing: the solve ended
      // with the panel product, and S_u exists only if an earlier solve of this linearisation built it
      s_valid = false;
      if (su_new) su_valid = false;
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
      // the rig members take the lead's pose increment mapped through D_j^-1 A_j D_lead, the group members the lead's f, k1, k2
      if (rig.n) TRY(rig_expand(D.inc, D.inc, false, 1));
      if (grp.n) TRY(group_expand(D.inc, D.inc, false));
    } else if (!have_inc) { g_err = "no device-resident increment (none solved since rba_linearize or rba_set_camera_fixed)"; return RBA_ERR_STATE; }
    int rc = start(ev_backsub); if (rc) return rc;
    CU(cudaMemsetAsync(d_flags, 0, 4 * sizeof(int), stream));
    const int grid = std::min(tile_grid(sm_count * 4), EBLOCKS);
    auto kb = D.lmp_slot ? k_back_substitute<S, true> : k_back_substitute<S>;  // + the landmark priors' part of l_diff
    kb<<<grid, TILE_WARPS * 32, 0, stream>>>(D, D.inc, d_epart, d_flags);
    k_sum_partials<1><<<1, 256, 0, stream>>>(d_epart, grid, d_red);
    launches += 2;
    rc = allreduce_scalars(1); if (rc) return rc;
    if (cprior.on) {  // the prior part of the model cost change, once, after the sum over the shards
      k_prior_ldiff<<<1, 256, 0, stream>>>(camera_prior(), D.inc, nc, d_red);
      ++launches;
    }
    if (pprior.n > 0) {  // the pair priors' part, likewise
      k_prior_ldiff<<<1, 256, 0, stream>>>(pair_prior(), D.inc, pprior.n, d_red);
      ++launches;
    }
    rc = stop(ev_backsub); if (rc) return rc;
    rc = start(ev_update); if (rc) return rc;
    if (update_cameras) {
      // NOTE: the reference skips the camera update when l_diff is not finite (linearizor_qr.cpp:275-277); the LM loop
      // then rejects the step and restores the backup, so updating unconditionally is equivalent for the caller.
      k_camera_update<S><<<(nc + 127) / 128, 128, 0, stream>>>(D, D.inc);
      ++launches;
      if (rig.n) TRY(rig_retie_state(D.cams));  // the members exactly at M_j T_lead: no drift over the iterations
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
    out->matvec_algorithmic_bytes = handover() == Handover::Assembled ? (81 * asm_nnzb + 18 * (int64_t)nc) * (int64_t)sizeof(S) + 4 * (asm_nnzb + nc + 1)
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
    TRY(matvec_launch(D.z, true));
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
    TRY(matvec_launch(D.p, false));  // warm-up
    TRY(start(ev_mv));
    for (int r = 0; r < reps; ++r) TRY(matvec_launch(D.p, false));
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
  bool asm_candidate() const { return asm_hook && opt.nranks == 1 && panels; }
  int setup_assembled() {
    if (!asm_candidate()) return RBA_OK;
    PairList P;
    const std::string msg = build_pair_list(L, P);
    if (!msg.empty()) { g_err = msg; return RBA_ERR_UNSUPPORTED; }
    // the product's deal is for the CTAs that are co-resident on an idle GPU
    int occ = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_rcs_spmv<S>, SPMV_CLASSES * 32, 0));
    AsmPlan A;
    const int ctas = std::max(1, occ) * sm_count;
    plan_assembled(L, P, sizeof(S), A, spmv_cap > 0 ? std::min(spmv_cap, ctas) : ctas);
    if (!A.fits) return RBA_OK;
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if ((size_t)A.device_bytes + ((size_t)256 << 20) > free_b) return RBA_OK;  // keep 256 MB for the rest of the handle and the caller
    TRY(upload(&d_asm_terms, A.terms));
    TRY(upload(&d_asm_wpos, P.wpos));
    TRY(upload(&d_asm_slots, P.terms));
    TRY(upload(&d_asm_blk_ptr, P.blk_ptr));
    TRY(upload(&d_asm_pos, A.pos));
    TRY(upload(&d_asm_col, A.col));
    TRY(upload(&d_spmv_chunks, A.spmv.chunks));
    TRY(upload(&d_spmv_chunk_ptr, A.spmv.chunk_ptr));
    spmv_grid = A.spmv.ctas;
    TRY(dalloc(&d_asm_stage, (size_t)A.nt * 81, false));
    TRY(dalloc(&d_asm_Su, (size_t)A.nblk * 81));
    TRY(dalloc(&d_asm_S, (size_t)A.nnzb * 81 + 16 / sizeof(S)));  // + 16 bytes: k_rcs_spmv's bulk copies round up
    asm_nt = A.nt; asm_nblk = (int)A.nblk; asm_nnzb = A.nnzb;
    asm_switch = asm_at > 0 ? asm_at : A.switch_iteration;
    asm_on = true;
    return RBA_OK;
  }
  // S_u (damping = 0: every term over the lambda-independent panel rows, staged and combined) or S = S_u + the damping
  // rows' part (damping = 1: from the dmp records of this solve's k_stage2, no staging; then the upper blocks)
  // (inside a solve only: all four kernels do nothing once its `done` flag is set.  They read it without a fence, which is
  // ordered only because they are plain stream launches after the vector step that sets it: not launched with PDL.)
  void assemble(int damping) {
    const int* done = &d_state->done;
    const unsigned per_entry = (unsigned)((81LL * asm_nblk + 255) / 256);
    if (damping) {
      k_rcs_damping<S><<<(asm_nblk + DMP_WARPS - 1) / DMP_WARPS, DMP_WARPS * 32, 0, stream>>>(
          d_asm_blk_ptr, (const int2*)d_asm_slots, asm_nblk, D.dmp, d_asm_Su, (const int2*)d_asm_pos, d_asm_S, done);
      k_rcs_mirror<S><<<per_entry, 256, 0, stream>>>((const int2*)d_asm_pos, asm_nblk, d_asm_S, done);
    } else {
      const int grid = (int)std::max<long long>(1, std::min<long long>((asm_nt + 23) / 24, (long long)sm_count * 16));
      k_rcs_terms<S><<<grid, 256, 0, stream>>>(D.panel, d_asm_terms, asm_nt, 0, d_asm_stage, done);
      k_rcs_combine<S><<<per_entry, 256, 0, stream>>>(d_asm_blk_ptr, d_asm_wpos, asm_nblk, d_asm_stage, d_asm_Su, done);
    }
    launches += 2;
  }

  // ------------------------------------------------------------------------------------------
  // Marginal covariances (DESIGN.md section 16).  Nothing of the handle changes: the scratch is allocated for the call and
  // freed before it returns; the state, the linearisation, the increment, the error cache and the timings are not touched.
  // The term lists (build_pair_list) built at the first call stay on the handle (not counted in device_bytes).
  int cov_build_lists() {
    if (cov_ready) return RBA_OK;
    PairList P;
    const std::string msg = build_pair_list(L, P);
    if (!msg.empty()) { g_err = msg; return RBA_ERR_UNSUPPORTED; }
    TRY(upload(&d_cov_blk_cam, P.blk_cam, false));
    TRY(upload(&d_cov_blk_ptr, P.blk_ptr, false));
    TRY(upload(&d_cov_terms, P.terms, false));
    TRY(upload(&d_cov_lm_slot0, P.slot0, false));
    TRY(upload(&d_cov_lm_n, P.nn, false));
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
  // P^T A P (expand = 0) or P A P^T (expand = 1) of the symmetric matrix whose lower triangle A holds, in place (full)
  int cov_group_passes(double* A, long long ld, long long n, int expand) {
    k_cov_group_symmetrize<<<dim3((unsigned)((n + 31) / 32), (unsigned)((n + 7) / 8)), dim3(32, 8), 0, stream>>>(A, ld, n);
    for (int columns = 0; columns < 2; ++columns)
      k_cov_group_pass<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(A, ld, n, groups(), columns, expand);
    CU(cudaGetLastError());
    return RBA_OK;
  }
  // P^T A P (expand = 0) or P A P^T (expand = 1) of the rigs' adjoint map, in place (full; DESIGN.md section 23)
  int cov_rig_passes(double* A, long long ld, long long n, int expand) {
    if (sen.n && !expand) TRY(sensor_tie());  // (sensors: M_j at the state the matrix is assembled at)
    k_cov_group_symmetrize<<<dim3((unsigned)((n + 31) / 32), (unsigned)((n + 7) / 8)), dim3(32, 8), 0, stream>>>(A, ld, n);
    for (int columns = 0; columns < 2; ++columns)
      if (sen.n)
        k_cov_rig_pass<S, true><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(A, ld, n, rigs(), columns, expand, sensors());
      else
        k_cov_rig_pass<S><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(A, ld, n, rigs(), columns, expand, NoSensors{});
    CU(cudaGetLastError());
    return RBA_OK;
  }
  // + the camera and pair priors' blocks (k_cov_priors) on the lower triangle of the unscaled matrix A (ld)
  void cov_priors(double* A, long long ld) {
    const bool prior_loss = cprior.loss.on || pprior.loss.on;
    if (cprior.on || pprior.n > 0)
      (prior_loss ? k_cov_priors<S, true> : k_cov_priors<S>)<<<(nc + 127) / 128, 128, 0, stream>>>(
          D.cams, nc, cprior.on ? cprior.mean.get() : nullptr, cprior.L.get(), pprior.ij.get(), pprior.mean.get(), pprior.L.get(),
          pprior.n > 0 ? pprior.ptr.get() : nullptr, pprior.item.get(), pprior.nbr.get(), A, ld,
          cprior.loss.on ? (const S*)cprior.loss.rec.get() : nullptr, pprior.loss.on ? (const S*)pprior.loss.rec.get() : nullptr, pprior.n);
  }
  // Cholesky of the lower triangle of the np x np matrix A (ld np) in place, right-looking by COV_TB tiles: factor the
  // diagonal tile, panel <- panel L_kk^-T, trailing lower tiles -= panel panel^T.  A pivot <= tau (or NaN) leaves the smallest
  // such index in *fail, on the device.  W [np][COV_TB] and Tt [COV_TB][COV_TB]: scratch.
  int dense_potrf(double* A, long long np, double* W, double* Tt, double tau, int* fail) {
    constexpr long long TB = COV_TB;
    const int nt = (int)(np / TB);
    for (int k = 0; k < nt; ++k) {
      const long long k0 = k * TB, m = np - k0 - TB;
      k_cov_tile_potrf<<<1, 256, 0, stream>>>(A, np, k0, tau, fail);
      if (m == 0) break;
      k_cov_tile_trtri<<<1, COV_TB, 0, stream>>>(A, np, k0, Tt, TB);
      double* P = A + (k0 + TB) + k0 * np;
      TRY(cov_copy(W, m, P, np, m, TB));
      cov_gemm<false, true>(m, TB, TB, 1.0, W, m, Tt, TB, 0.0, P, np, 0, 0);
      cov_gemm<false, true>(m, m, TB, -1.0, P, np, P, np, 1.0, P + TB * np, np, 1, 0);
    }
    return RBA_OK;
  }

  // ------------------------------------------------------------------------------------------
  // preconditioner_type = CLUSTER_JACOBI (cluster_precond.cuh, DESIGN.md section 28)
  // The per-solve vectors and the default clustering (rba_cluster_cameras with RBA_CLUSTER_DEFAULT_CAMERAS).
  int setup_clusters(const rba_problem_view* pv) {
    if (opt.preconditioner_type != 2) return RBA_OK;
    clu.dflt.resize((size_t)nc);
    const std::string msg = cluster_cameras(nc, nl_total, pv->lm_obs_offset, pv->obs_cam_idx, RBA_CLUSTER_DEFAULT_CAMERAS, clu.dflt.data());
    if (!msg.empty()) { g_err = msg; return RBA_ERR_INVALID_ARGUMENT; }
    for (S** v : {&clu.bh, &clu.w, &clu.yh}) TRY(dalloc(v, (size_t)9 * nc));
    TRY(dalloc(&clu.eye, (size_t)81 * nc));
    clu.on = true;
    return set_camera_clusters(nullptr);
  }
  // Every check runs before anything changes, and the new buffers are adopted once they all exist, so a rejected or failed
  // call leaves the previous clustering.
  int set_camera_clusters(const int32_t* cluster_of) override {
    if (!clu.on) { g_err = "rba_set_camera_clusters: the handle's preconditioner_type is not CLUSTER_JACOBI"; return RBA_ERR_STATE; }
    std::vector<int> host = cluster_of ? std::vector<int>(cluster_of, cluster_of + nc) : clu.dflt;
    ClusterPlan P;
    const std::string msg = plan_clusters(L, host.data(), panels, P);
    if (!msg.empty()) { g_err = "rba_set_camera_clusters: " + msg; return RBA_ERR_INVALID_ARGUMENT; }
    ClusterTerm next;
    TRY(fit(next.ptr, {}, P.ptr.size(), &P.ptr)); TRY(fit(next.cams, {}, P.cams.size(), &P.cams));
    TRY(fit(next.xb_ptr, {}, P.xb_ptr.size(), &P.xb_ptr)); TRY(fit(next.blk_off, {}, P.blk_off.size(), &P.blk_off));
    TRY(fit(next.fac_off, {}, P.fac_off.size(), &P.fac_off)); TRY(fit(next.xb, {}, P.xb.size(), &P.xb));
    TRY(fit(next.slots, {}, P.slots.size(), &P.slots)); TRY(fit(next.panel_terms, {}, P.panel_terms.size(), &P.panel_terms));
    TRY(alloc(next.status, (size_t)P.ncl, true)); TRY(alloc(next.blocks, (size_t)P.blk_off[P.ncl], true));
    TRY(alloc(next.factor, (size_t)P.fac_off[P.ncl], true));
    const size_t smem = (size_t)81 * P.max_k * P.max_k * sizeof(double), fsmem = cluster_factor_smem(P.max_k);
    CU(cudaFuncSetAttribute(k_cluster_build<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CU(cudaFuncSetAttribute(k_cluster_fwd<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    CU(cudaFuncSetAttribute(k_cluster_back<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    CU(cudaStreamSynchronize(stream));
    clu.adopt(next);
    clu.host = std::move(host);
    clu.ncl = P.ncl; clu.max_k = P.max_k; clu.blk_n = P.blk_off[P.ncl]; clu.fac_n = P.fac_off[P.ncl];
    clu.built = false;
    return RBA_OK;
  }
  static size_t cluster_factor_smem(int max_k) { return (size_t)(9 * max_k) * (9 * max_k + 1) / 2 * sizeof(double); }
  ClusterView cluster_view() const {
    return {clu.ncl, clu.ptr.get(), clu.cams.get(), clu.blk_off.get(), clu.fac_off.get(), clu.xb_ptr.get(), clu.xb.get(),
            (const int2*)clu.slots.get(), panels ? clu.panel_terms.get() : nullptr, clu.blocks.get(), clu.factor.get(), clu.status.get()};
  }
  // the cluster blocks of this solve's lambda, their factors, the vector step's identity blocks and bh = L^-1 b (after
  // k_precond_invert: the SCHUR_JACOBI blocks are written and b is final)
  int cluster_build() {
    const ClusterView cv = cluster_view();
    k_cluster_build<S><<<clu.ncl, 256, (size_t)81 * clu.max_k * clu.max_k * sizeof(double), stream>>>(cv, D, clu.eye);
    k_cluster_fwd<S><<<clu.ncl, CLUSTER_THREADS, cluster_factor_smem(clu.max_k), stream>>>(cv, D, D.b, nullptr, nullptr, S(0), clu.bh, nullptr);
    launches += 2;
    clu.built = true;
    return RBA_OK;
  }
  // y = L^-T v (done: inside a solve, nothing once it has ended)
  void cluster_back(const S* v, S* y, const int* done) {
    k_cluster_back<S><<<clu.ncl, CLUSTER_THREADS, cluster_factor_smem(clu.max_k), stream>>>(cluster_view(), v, y, done);
    ++launches;
  }
  int get_cluster_precond(int32_t* cluster_of, double* blocks, int32_t* status) override {
    if (!clu.on) { g_err = "rba_get_cluster_preconditioner: the handle's preconditioner_type is not CLUSTER_JACOBI"; return RBA_ERR_STATE; }
    if ((blocks || status) && !clu.built) { g_err = "rba_get_cluster_preconditioner: no solve has assembled the blocks of this clustering"; return RBA_ERR_STATE; }
    if (cluster_of) std::copy(clu.host.begin(), clu.host.end(), cluster_of);
    if (blocks) CU(cudaMemcpyAsync(blocks, clu.blocks.get(), (size_t)clu.blk_n * sizeof(double), cudaMemcpyDeviceToHost, stream));
    if (status) CU(cudaMemcpyAsync(status, clu.status.get(), (size_t)clu.ncl * sizeof(int), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return RBA_OK;
  }

  // ------------------------------------------------------------------------------------------
  // linear_solver_type = DENSE_SCHUR (dense_solve.cuh, DESIGN.md section 27)
  // the bytes setup_dense allocates: A, W, Tt, d, x, y, the per-slot rows and the pivot flag
  void dense_bytes(long long& np, size_t& total) const {
    np = (9LL * nc + COV_TB - 1) / COV_TB * COV_TB;
    const size_t ns = (size_t)L.nslots;
    total = (size_t)(np * np + np * COV_TB + COV_TB * COV_TB + 3 * np) * 8 + ns * (18 + 27) * 8 + 4;
  }
  // Everything a solve uses, allocated once and counted in device_bytes: the matrix, the potrf scratch, the vectors, the
  // per-slot rows and the term lists of the covariances (build_pair_list).
  int setup_dense() {
    if (opt.linear_solver_type != 1) return RBA_OK;
    long long np = 0;
    size_t total = 0;
    dense_bytes(np, total);
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (total > free_b) {
      g_err = "DENSE_SCHUR needs " + std::to_string(total) + " bytes of device memory (a dense " + std::to_string(np) + " x " +
              std::to_string(np) + " float64 reduced camera matrix plus scratch); " + std::to_string(free_b) + " bytes are free";
      return RBA_ERR_UNSUPPORTED;
    }
    TRY(cov_build_lists());
    TRY(dalloc(&dn.A, (size_t)(np * np), false));
    TRY(dalloc(&dn.W, (size_t)(np * COV_TB), false));
    TRY(dalloc(&dn.Tt, (size_t)(COV_TB * COV_TB), false));
    TRY(dalloc(&dn.d, (size_t)np, false));
    TRY(dalloc(&dn.x, (size_t)np, false));
    TRY(dalloc(&dn.y, (size_t)np, false));
    TRY(dalloc(&dn.jp, (size_t)L.nslots * 18, false));
    TRY(dalloc(&dn.kb, (size_t)L.nslots * 27, false));
    TRY(dalloc(&dn.fail, 1, false));
    dn.np = np;
    return RBA_OK;
  }
  // The exact increment of the system PCG iterates on, after stage 2 and the preconditioner of this solve: no host
  // synchronisation, the pivot flag is read on the device by k_dense_finish.
  int dense_enqueue(double lambda, void* inc_out) {
    TRY(start(ev_pcg));
    constexpr long long TB = COV_TB;
    const long long n = 9LL * nc, np = dn.np;
    const int nl = L.nl_local, nt = (int)(np / TB);
    const uint8_t* held = grp.n || rig.n ? tied_fixed() : D.cam_fixed;
    double* A = dn.A;
    CU(cudaMemsetAsync(A, 0, (size_t)(np * np) * 8, stream));
    CU(cudaMemsetAsync(dn.fail, 0x7f, 4, stream));
    CU(cudaMemsetAsync(d_state, 0, sizeof(PcgState), stream));
    // 1.-2. the damped elimination, assembly, priors, ties, scaling, held parameters, lambda
    k_dense_landmark<S><<<std::max(1, std::min((nl + 3) / 4, sm_count * 16)), 128, 0, stream>>>(
        D, ko, d_cov_lm_slot0, d_cov_lm_n, nl, lambda, dn.jp, dn.kb, lprior.n > 0 ? lprior.of_lm.get() : nullptr);
    k_cov_assemble<<<std::max(1, std::min((cov_nblk + 7) / 8, sm_count * 8)), 256, 0, stream>>>(
        (const int2*)d_cov_blk_cam, d_cov_blk_ptr, (const int2*)d_cov_terms, cov_nblk, dn.jp, dn.kb, A, np);
    launches += 2 + ((cprior.on || pprior.n > 0) ? 1 : 0);
    cov_priors(A, np);
    if (rig.n) { TRY(cov_rig_passes(A, np, n, 0)); launches += 3; }
    if (grp.n) { TRY(cov_group_passes(A, np, n, 0)); launches += 3; }
    const unsigned g1 = (unsigned)((np + 255) / 256);
    k_dense_scaling<S><<<g1, 256, 0, stream>>>(D.scaling, n, np, dn.d);
    if (rig.n) {
      k_dense_tied_scaling<S><<<(rig.n + sen.n + 127) / 128, 128, 0, stream>>>(rigs(), sen.ds.get(), sen.ptr.get(), sen.mem.get(), sen.n, dn.d);
      ++launches;
    }
    k_cov_equil<<<dim3((unsigned)(np / 32), (unsigned)(np / 8)), dim3(32, 8), 0, stream>>>(A, np, n, np, held, dn.d);
    k_dense_gather<S><<<g1, 256, 0, stream>>>(A, np, n, np, held, lambda, D.b, dn.x, dn.fail);
    launches += 3;
    // 3. potrf: 4 kernels per tile but the last
    TRY(dense_potrf(A, np, dn.W, dn.Tt, 0.0, dn.fail));
    launches += 4LL * nt - 3;
    // 4. L y = b, L^T x = y
    for (int k = 0; k < nt; ++k) {
      const long long k0 = k * TB, m = np - k0 - TB;
      k_dense_trsv_fwd<<<(unsigned)std::max(1LL, (m + DENSE_TRSV_ROWS - 1) / DENSE_TRSV_ROWS), DENSE_TRSV_ROWS, 0, stream>>>(A, np, np, k0,
                                                                                                                          dn.x, dn.y);
    }
    for (int k = nt - 1; k >= 0; --k) {
      const long long k0 = k * TB;
      k_dense_trsv_bwd<<<(unsigned)std::max(1LL, (k0 + DENSE_TRSV_COLS - 1) / DENSE_TRSV_COLS), 256, 0, stream>>>(A, np, k0, dn.y, dn.x);
    }
    // 5. the increment and the summary
    k_dense_finish<S><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dn.x, n, np, held, dn.fail, D.inc, d_state);
    launches += 2LL * nt + 1;
    CU(cudaGetLastError());
    TRY(tie_expand(D.inc));  // inc = P u for the back-substitution, the update and inc_out
    CU(cudaMemcpyAsync(&h_state[0], d_state, sizeof(PcgState), cudaMemcpyDeviceToHost, stream));
    if (inc_out) CU(cudaMemcpyAsync(inc_out, D.inc, (size_t)9 * nc * sizeof(S), cudaMemcpyDeviceToHost, stream));
    TRY(stop(ev_pcg));
    have_inc = true;
    new_linearization_point = false;
    return RBA_OK;
  }
  // The dense inverse of one covariance call and what its extraction kernels read; the scratch is freed (after the kernels
  // have finished: cudaFree waits for them) when it goes out of scope.
  struct CovInverse {
    DeviceBuffer<char> scratch;
    double* A = nullptr;  // S_eq^-1 (lower triangle, leading dimension np); cov_sinv reads D S_eq^-1 D from it
    double* d = nullptr;  // the diagonal of D
    double* kb = nullptr; double* wl = nullptr; int* rk = nullptr;  // K per slot, W and rank per landmark
    long long np = 0;
  };
  // Steps 1-3 of DESIGN.md section 16, shared by rba_compute_covariance and rba_compute_covariance_blocks (`fn` names the entry
  // point in the messages).  One device allocation holds the pipeline's scratch followed by the caller's buffers of `extra`
  // bytes each (their addresses are returned in `out`); the byte count of the out-of-memory message includes them.
  int cov_factor_inverse(const char* fn, const std::vector<size_t>& extra, CovInverse& c, std::vector<char*>& out) {
    if (opt.nranks > 1) {
      g_err = std::string(fn) + ": sharded handles (nranks > 1) are not supported: the reduced camera matrix would need a cross-rank sum";
      return RBA_ERR_UNSUPPORTED;
    }
    TRY(cov_build_lists());
    constexpr long long TB = COV_TB;
    const long long n = 9LL * nc, np = (n + TB - 1) / TB * TB, ns = L.nslots;
    const int nl = L.nl_local, nt = (int)(np / TB), n_lmp = lprior.n;
    size_t total = 0;
    auto carve = [&](size_t bytes) { const size_t o = total; total += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_A = carve((size_t)(np * np) * 8), o_W = carve((size_t)(np * TB) * 8), o_Y = carve((size_t)(np * TB) * 8),
                 o_T = carve((size_t)(TB * TB) * 8), o_d = carve((size_t)np * 8), o_jp = carve((size_t)ns * 18 * 8),
                 o_kb = carve((size_t)ns * 27 * 8), o_wl = carve((size_t)nl * 9 * 8), o_rk = carve((size_t)nl * 4), o_fail = carve(4);
    std::vector<size_t> o_extra;
    for (size_t b : extra) o_extra.push_back(carve(b));
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (total > free_b) {
      g_err = std::string(fn) + " needs " + std::to_string(total) + " bytes of device memory (a dense " + std::to_string(n) + " x " +
              std::to_string(n) + " float64 reduced camera matrix plus scratch); " + std::to_string(free_b) + " bytes are free";
      return RBA_ERR_UNSUPPORTED;
    }
    TRY(alloc(c.scratch, total, false, false));
    char* base = c.scratch.get();
    double* A = (double*)(base + o_A); double* W = (double*)(base + o_W); double* Y = (double*)(base + o_Y);
    double* Tt = (double*)(base + o_T); double* d = (double*)(base + o_d); double* jp = (double*)(base + o_jp);
    double* kb = (double*)(base + o_kb); double* wl = (double*)(base + o_wl); int* rk = (int*)(base + o_rk);
    int* fail = (int*)(base + o_fail);
    out.clear();
    for (size_t o : o_extra) out.push_back(base + o);
    const int wgrid = std::max(1, std::min((nl + 3) / 4, sm_count * 16));
    c.A = A; c.d = d; c.kb = kb; c.wl = wl; c.rk = rk; c.np = np;
    // 1.-2. elimination, assembly, priors, held parameters, equilibration
    CU(cudaMemsetAsync(A, 0, (size_t)(np * np) * 8, stream));
    CU(cudaMemsetAsync(fail, 0x7f, 4, stream));
    // LMP: + L^T L of the landmark priors in Hll; OBSW: the rows whitened by the observation information; OBSL: the
    // observations' own losses
    auto kcov = n_lmp > 0 ? (D.obs_W ? k_cov_landmark<S, true, true> : k_cov_landmark<S, true>)
                          : (D.obs_W ? k_cov_landmark<S, false, true> : k_cov_landmark<S>);
    if (D.obs_loss) kcov = n_lmp > 0 ? kcov_of<true>(D.obs_W, true) : kcov_of<false>(D.obs_W, true);
    if (lprior.loss.on) kcov = kcov_lmpl(D.obs_W, D.obs_loss);  // LMPL: the landmark priors' losses (section 22)
    kcov<<<wgrid, 128, 0, stream>>>(D, ko, d_cov_lm_slot0, d_cov_lm_n, nl, jp, kb, wl, rk, n_lmp > 0 ? lprior.of_lm.get() : nullptr);
    k_cov_assemble<<<std::max(1, std::min((cov_nblk + 7) / 8, sm_count * 8)), 256, 0, stream>>>(
        (const int2*)d_cov_blk_cam, d_cov_blk_ptr, (const int2*)d_cov_terms, cov_nblk, jp, kb, A, np);
    // LOSS: the camera and pair priors' losses (section 22), their weights re-evaluated in double at the current state
    cov_priors(A, np);
    // intrinsics groups (DESIGN.md section 18): S_u = P^T S P, the members' entries 6..8 then held like the user's
    // (rigs, section 23: S_u = P^T S P through the adjoints, the members' pose entries then held)
    const uint8_t* held = D.cam_fixed;
    if (rig.n) TRY(cov_rig_passes(A, np, n, 0));
    if (grp.n) TRY(cov_group_passes(A, np, n, 0));
    if (grp.n || rig.n) held = tied_fixed();
    k_cov_diag<<<(unsigned)((np + 255) / 256), 256, 0, stream>>>(A, np, n, np, held, d);
    k_cov_equil<<<dim3((unsigned)(np / 32), (unsigned)(np / 8)), dim3(32, 8), 0, stream>>>(A, np, n, np, held, d);
    TRY(dense_potrf(A, np, W, Tt, COV_PIVOT_TAU, fail));
    int h_fail = 0;
    CU(cudaMemcpyAsync(&h_fail, fail, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    CU(cudaGetLastError());
    if (h_fail < n) {
      static const char* names[9] = {"tx", "ty", "tz", "rx", "ry", "rz", "f", "k1", "k2"};
      g_err = std::string(fn) + ": the reduced camera matrix is singular: Cholesky pivot <= " + std::to_string(COV_PIVOT_TAU) +
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
    // (rigs: the inverse un-equilibrated, then P S_u^-1 P^T through the adjoints with a unit equilibration)
    if (rig.n) {
      k_cov_group_symmetrize<<<dim3((unsigned)((n + 31) / 32), (unsigned)((n + 7) / 8)), dim3(32, 8), 0, stream>>>(A, np, n);
      k_cov_unequil<<<dim3((unsigned)((n + 31) / 32), (unsigned)((n + 7) / 8)), dim3(32, 8), 0, stream>>>(A, np, n, d);
      k_cov_unit_d<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d, n);
      TRY(cov_rig_passes(A, np, n, 1));
    }
    // (intrinsics groups: P S_u^-1 P^T, the members' rows and columns 6..8 and equilibration those of the lead)
    if (grp.n) {
      TRY(cov_group_passes(A, np, n, 1));
      k_cov_group_d<<<1, 1, 0, stream>>>(d, groups());
    }
    return RBA_OK;
  }
  // The request kinds of an rba_covariance_query in the order of its fields: the ranges of a request's indices (a, b) and
  // the doubles of its block.
  struct CovKind { const char* name; int m; const int32_t* req; double* out; int lim0, lim1, width; };
  std::array<CovKind, 4> cov_kinds(const rba_covariance_query& q) const {
    return {{{"camera_pairs", q.num_camera_pairs, q.camera_pairs, q.camera_cross, nc, nc, 81},
             {"camera_landmark", q.num_camera_landmark, q.camera_landmark, q.camera_landmark_cross, nc, nl_total, 27},
             {"landmark_pairs", q.num_landmark_pairs, q.landmark_pairs, q.landmark_cross, nl_total, nl_total, 9},
             {"relative_pairs", q.num_relative_poses, q.relative_pairs, q.relative_cov, nc, nc, 36}}};
  }
  int compute_covariance(double* cam_cov, double* lm_cov) override {
    if (!cam_cov && !lm_cov) { g_err = "rba_compute_covariance: cam_cov and lm_cov are both NULL"; return RBA_ERR_INVALID_ARGUMENT; }
    rba_covariance_query q = {};
    q.cam_cov = cam_cov;
    q.lm_cov = lm_cov;
    return cov_compute("rba_compute_covariance", q);
  }
  // Covariance blocks of chosen pairs (DESIGN.md section 20): every request is checked before any device work.
  int compute_covariance_blocks(const rba_covariance_query* q) override {
    auto bad = [](const std::string& m) { g_err = "rba_compute_covariance_blocks: " + m; return RBA_ERR_INVALID_ARGUMENT; };
    if (!q) return bad("q is NULL");
    const std::array<CovKind, 4> kinds = cov_kinds(*q);
    bool any = q->cam_cov || q->lm_cov;
    for (int k = 0; k < 4; ++k) {
      const CovKind& K = kinds[k];
      if (K.m < 0) return bad(std::string("num_") + K.name + " is negative");
      if (K.m == 0) continue;
      any = true;
      if (!K.req || !K.out) return bad(std::string(K.name) + " or its output is NULL with a positive count");
      for (int r = 0; r < K.m; ++r) {
        const int32_t a = K.req[2 * r], b = K.req[2 * r + 1];
        if (a < 0 || a >= K.lim0 || b < 0 || b >= K.lim1)
          return bad(std::string(K.name) + " request " + std::to_string(r) + " (" + std::to_string(a) + ", " + std::to_string(b) +
                     ") is out of range");
        if (k == 3 && a == b) return bad("relative_pairs request " + std::to_string(r) + " has i == j");
      }
    }
    if (!any) return bad("nothing is requested (all counts are 0 and cam_cov and lm_cov are NULL)");
    return cov_compute("rba_compute_covariance_blocks", *q);
  }
  // One covariance call on a query its entry point `fn` (named in the messages) has checked: cov_factor_inverse, then the
  // extraction kernels.  The marginals cam_cov and lm_cov are the diagonal requests (k, k) of k_cov_cam_cross and
  // k_cov_lm_cross (req == nullptr, no request list).  Output space is carved only for what is asked for; the requests are
  // copied into the call's scratch and the outputs copied back at the end.
  int cov_compute(const char* fn, const rba_covariance_query& q) {
    const int nl = L.nl_local;
    const std::array<CovKind, 4> kinds = cov_kinds(q);
    std::vector<size_t> extra = {q.cam_cov ? (size_t)nc * 81 * 8 : 0, q.lm_cov ? (size_t)nl * 9 * 8 : 0};
    for (const CovKind& K : kinds) {
      extra.push_back((size_t)K.m * 8);
      extra.push_back((size_t)K.m * K.width * 8);
    }
    CovInverse c;
    std::vector<char*> buf;
    TRY(cov_factor_inverse(fn, extra, c, buf));
    const int2* req[4];
    double* dout[4];
    for (int k = 0; k < 4; ++k) {
      req[k] = (const int2*)buf[2 + 2 * k];
      dout[k] = (double*)buf[3 + 2 * k];
      if (kinds[k].m > 0)
        CU(cudaMemcpyAsync(buf[2 + 2 * k], kinds[k].req, (size_t)kinds[k].m * 8, cudaMemcpyHostToDevice, stream));
    }
    const auto grid = [&](long long items, int per_block) {
      return (unsigned)std::max<long long>(1, std::min<long long>((items + per_block - 1) / per_block, (long long)sm_count * 16));
    };
    const auto cam_cross = [&](const int2* r, int m, double* out) {
      k_cov_cam_cross<<<grid(81LL * m, 256), 256, 0, stream>>>(c.A, c.np, c.d, D.cam_fixed, r, m, out);
    };
    const auto lm_cross = [&](const int2* r, int m, double* out) {
      (r ? k_cov_lm_cross<false> : k_cov_lm_cross<true>)<<<grid(m, 4), 128, 0, stream>>>(
          c.A, c.np, c.d, D.cam_fixed, D.slot_cam, d_cov_lm_slot0, d_cov_lm_n, c.kb, c.wl, c.rk, r, m, out);
    };
    if (q.cam_cov) cam_cross(nullptr, nc, (double*)buf[0]);
    if (q.lm_cov) lm_cross(nullptr, nl, (double*)buf[1]);
    if (kinds[0].m > 0) cam_cross(req[0], kinds[0].m, dout[0]);
    if (kinds[1].m > 0)
      k_cov_cam_lm<<<grid(kinds[1].m, 4), 128, 0, stream>>>(c.A, c.np, c.d, D.cam_fixed, D.slot_cam, d_cov_lm_slot0, d_cov_lm_n, c.kb,
                                                            c.wl, c.rk, req[1], kinds[1].m, dout[1]);
    if (kinds[2].m > 0) lm_cross(req[2], kinds[2].m, dout[2]);
    if (kinds[3].m > 0)
      k_cov_rel_pose<S><<<grid(kinds[3].m, COV_REL_THREADS), COV_REL_THREADS, 0, stream>>>(c.A, c.np, c.d, D.cam_fixed, D.cams, req[3],
                                                                                         kinds[3].m, dout[3]);
    if (q.cam_cov) CU(cudaMemcpyAsync(q.cam_cov, buf[0], (size_t)nc * 81 * 8, cudaMemcpyDeviceToHost, stream));
    if (q.lm_cov) CU(cudaMemcpyAsync(q.lm_cov, buf[1], (size_t)nl * 9 * 8, cudaMemcpyDeviceToHost, stream));
    for (int k = 0; k < 4; ++k)
      if (kinds[k].m > 0)
        CU(cudaMemcpyAsync(kinds[k].out, dout[k], (size_t)kinds[k].m * kinds[k].width * 8, cudaMemcpyDeviceToHost, stream));
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
int32_t rba_set_intrinsics_groups(rba_handle* h, const int32_t* group) { return h->set_intrinsics_groups(group); }
int32_t rba_set_camera_rigs(rba_handle* h, const int32_t* rig, const void* cam_from_rig) { return h->set_camera_rigs(rig, cam_from_rig); }
int32_t rba_set_rig_sensors(rba_handle* h, const int32_t* sensor) { return h->set_rig_sensors(sensor); }
int32_t rba_get_rig_extrinsics(rba_handle* h, void* cam_from_rig) { return h->get_rig_extrinsics(cam_from_rig); }
int32_t rba_set_observation_info(rba_handle* h, const void* sqrt_info) { return h->set_observation_info(sqrt_info); }
int32_t rba_set_observation_loss(rba_handle* h, const uint8_t* kind, const void* scale) { return h->set_observation_loss(kind, scale); }
int32_t rba_set_prior_loss(rba_handle* h, int32_t prior_kind, int32_t num, const uint8_t* kind, const void* scale) {
  return h->set_prior_loss(prior_kind, num, kind, scale);
}
int32_t rba_get_prior_residuals(rba_handle* h, int32_t prior_kind, void* residual, void* robust_weight) {
  return h->get_prior_residuals(prior_kind, residual, robust_weight);
}
void rba_default_triangulate_opts(rba_triangulate_opts* o) {
  *o = rba_triangulate_opts{};
  o->mode = RBA_TRIANGULATE_LINEAR | RBA_TRIANGULATE_REFINE;
  o->max_iterations = 20;
  o->min_angle = 0.0;
  o->function_tolerance = 1e-10;
}
int32_t rba_triangulate_landmarks(rba_handle* h, const rba_triangulate_opts* o, int32_t num, const int32_t* lm_idx,
                                  uint8_t* status, double* angle, double* cost) {
  return h->triangulate(o, num, lm_idx, status, angle, cost);
}
void rba_default_resect_opts(rba_resect_opts* o) {
  *o = rba_resect_opts{};
  o->mode = RBA_RESECT_LINEAR | RBA_RESECT_REFINE;
  o->max_iterations = 20;
  o->function_tolerance = 1e-10;
}
int32_t rba_resect_cameras(rba_handle* h, const rba_resect_opts* o, int32_t num, const int32_t* cam_idx, uint8_t* status,
                           int32_t* points, double* cost) {
  return h->resect(o, num, cam_idx, status, points, cost);
}
int32_t rba_get_observation_residuals(rba_handle* h, void* residual, void* robust_weight, uint8_t* flags) {
  return h->get_observation_residuals(residual, robust_weight, flags);
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
int32_t rba_cluster_cameras(const rba_problem_view* p, int32_t max_cluster_size, int32_t* cluster_of_camera) {
  if (!p || !cluster_of_camera || p->num_cameras <= 0 || p->num_landmarks < 0 || !p->lm_obs_offset || (p->num_landmarks > 0 && !p->obs_cam_idx)) {
    rba::g_err = "rba_cluster_cameras: null or empty argument";
    return RBA_ERR_INVALID_ARGUMENT;
  }
  const std::string msg = rba::cluster_cameras(p->num_cameras, p->num_landmarks, p->lm_obs_offset, p->obs_cam_idx, max_cluster_size,
                                               cluster_of_camera);
  if (!msg.empty()) { rba::g_err = "rba_cluster_cameras: " + msg; return RBA_ERR_INVALID_ARGUMENT; }
  return RBA_OK;
}
int32_t rba_set_camera_clusters(rba_handle* h, const int32_t* cluster_of_camera) { return h->set_camera_clusters(cluster_of_camera); }
int32_t rba_get_cluster_preconditioner(rba_handle* h, int32_t* cluster_of_camera, double* blocks, int32_t* status) {
  return h->get_cluster_precond(cluster_of_camera, blocks, status);
}
int32_t rba_right_multiply(rba_handle* h, const void* x, void* y) { return h->right_multiply(x, y); }
int32_t rba_debug_get_block(rba_handle* h, int32_t lm, void* out, int32_t rows, int32_t cols, void* jls) {
  return h->debug_get_block(lm, out, rows, cols, jls);
}
int32_t rba_compute_covariance(rba_handle* h, double* cam_cov, double* lm_cov) { return h->compute_covariance(cam_cov, lm_cov); }
int32_t rba_compute_covariance_blocks(rba_handle* h, const rba_covariance_query* q) { return h->compute_covariance_blocks(q); }
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
