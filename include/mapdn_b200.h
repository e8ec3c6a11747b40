/*
 * mapdn_b200.h - C-ABI of the H100-native batched MAPDN voltage-control environment step.
 *
 * The reference (Future-Power-Networks/MAPDN) has no FFI: the hot path sits behind the Python
 * class VoltageControl(MultiAgentEnv) (environments/var_voltage_control/voltage_control_env.py)
 * which calls the third-party pandapower.runpp once per env per step (:124, :165, :557).
 * This header is the boundary a replacement binds instead (ctypes stub: INTEGRATION.md;
 * in-tree binding: mapdn_b200/_capi.py). Plain pointers and sizes only - no torch types.
 *
 * Conventions
 *  - every function returns mapdn_status (0 = OK); never throws; mapdn_last_error() gives text.
 *  - "dev" pointers are device memory on the handle's GPU, caller-owned, row-major [B, n],
 *    fp64 unless noted. "host" pointers are host memory (pinned for async copies).
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream). Calls are
 *    stream-ordered and do not synchronise the host unless documented (the *_host entry points
 *    synchronise `stream` before returning).
 *  - Solver divergence is DATA, not an error: per-env converged/destroy flags
 *    (reference :188-196,204).
 *  - A handle is bound to one device and is not thread-safe.
 */
#ifndef MAPDN_B200_H
#define MAPDN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MAPDN_ABI_VERSION 2
#define MAPDN_N_INFO 11   /* info dict keys, reference :585-606,621 (order: mapdn_info_key) */

typedef enum {
  MAPDN_OK = 0,
  MAPDN_ERR_INVALID = 1,      /* bad argument / inconsistent description               */
  MAPDN_ERR_CUDA = 2,         /* CUDA runtime failure (text in mapdn_last_error)       */
  MAPDN_ERR_TOPOLOGY = 3,     /* not connected, or meshed with more than 256 PQ buses  */
  MAPDN_ERR_UNSUPPORTED = 4,  /* feature of the reference not implemented              */
  MAPDN_ERR_NOMEM = 5
} mapdn_status;

/* reference voltage_barrier/voltage_barrier_registry.py:9-15 */
typedef enum {
  MAPDN_BARRIER_L1 = 0, MAPDN_BARRIER_L2 = 1, MAPDN_BARRIER_BOWL = 2,
  MAPDN_BARRIER_BUMP = 3, MAPDN_BARRIER_COURANT_BELTRAMI = 4
} mapdn_barrier;

/* order of the 11 floats in info[B, 11] (reference _calc_reward :585-606,621) */
typedef enum {
  MAPDN_INFO_PCT_V_OUT = 0, MAPDN_INFO_PCT_V_LOW = 1, MAPDN_INFO_PCT_V_HIGH = 2,
  MAPDN_INFO_TOTALLY_CONTROLLABLE = 3, MAPDN_INFO_AVG_V_DEV = 4, MAPDN_INFO_AVG_V = 5,
  MAPDN_INFO_MAX_V_DROP_DEV = 6, MAPDN_INFO_MAX_V_RISE_DEV = 7, MAPDN_INFO_TOTAL_LINE_LOSS = 8,
  MAPDN_INFO_Q_LOSS = 9, MAPDN_INFO_DESTROY = 10
} mapdn_info_key;

/* per-env result columns readable with mapdn_get_field (reference tester getters :625-647) */
typedef enum {
  MAPDN_FIELD_VM = 0,        /* res_bus.vm_pu      [B, n_bus]   (_get_res_bus_v)        */
  MAPDN_FIELD_VA_DEG = 1,    /* res_bus.va_degree  [B, n_bus]                           */
  MAPDN_FIELD_P_BUS = 2,     /* res_bus.p_mw       [B, n_bus]   (_get_res_bus_active)   */
  MAPDN_FIELD_Q_BUS = 3,     /* res_bus.q_mvar     [B, n_bus]   (_get_res_bus_reactive) */
  MAPDN_FIELD_P_SGEN = 4,    /* sgen.p_mw          [B, n_sgen]  (_get_sgen_active)      */
  MAPDN_FIELD_Q_SGEN = 5,    /* sgen.q_mvar        [B, n_sgen]  (_get_sgen_reactive)    */
  MAPDN_FIELD_LINE_LOSS = 6, /* res_line.pl_mw     [B, n_line]  (_get_res_line_loss)    */
  MAPDN_FIELD_P_LOAD = 7,    /* load.p_mw          [B, n_load]                          */
  MAPDN_FIELD_Q_LOAD = 8,    /* load.q_mvar        [B, n_load]                          */
  MAPDN_FIELD_SUM_REWARDS = 9, /* self.sum_rewards [B]                                  */
  MAPDN_FIELD_STEPS = 10,    /* self.steps as fp64 [B]                                  */
  MAPDN_FIELD_START_ROW = 11,/* episode window start row as fp64 [B]                    */
  MAPDN_FIELD_NR_ITERS = 12  /* Newton iterations of the last power flow as fp64 [B]    */
                             /* (max_iter when it diverged; SURVEY 8d side metric)      */
} mapdn_field;

/*
 * Static network, per-unit on base_mva - what pandapower's _pd2ppc produces from model.p
 * (replaces reference _load_network :400-405 + the per-call conversion inside pp.runpp).
 * Buses 0..n_bus-1 in ascending pandapower bus index. All arrays are HOST memory, copied.
 * Optional arrays may be NULL (defaults in brackets).
 */
typedef struct {
  int32_t n_bus, n_branch, n_load, n_sgen;
  double base_mva;            /* net.sn_mva                                             */
  int32_t slack_bus;          /* bus of the single ext_grid                             */
  double slack_vm;            /* ext_grid.vm_pu                                         */
  double slack_va_deg;        /* ext_grid.va_degree                                     */
  double vm_init;             /* flat-start |V| of PQ buses (pandapower init="auto")    */
  const int32_t* br_from;     /* [n_branch]                                             */
  const int32_t* br_to;       /* [n_branch]                                             */
  const double* br_r;         /* [n_branch] series resistance p.u.                      */
  const double* br_x;         /* [n_branch] series reactance p.u.                       */
  const double* br_b;         /* [n_branch] total charging susceptance p.u. [0]         */
  const double* br_g;         /* [n_branch] total shunt conductance p.u.    [0]         */
  const double* br_tap;       /* [n_branch] off-nominal ratio, 0 => 1       [1]         */
  const double* br_shift_deg; /* [n_branch] phase shift                     [0]         */
  const uint8_t* br_status;   /* [n_branch] in service                      [1]         */
  const uint8_t* br_is_line;  /* [n_branch] row appears in res_line         [1]         */
  const double* bus_gs_mw;    /* [n_bus] shunt P at 1 p.u.                  [0]         */
  const double* bus_bs_mvar;  /* [n_bus] shunt Q injection at 1 p.u.        [0]         */
  const int32_t* bus_zone;    /* [n_bus] zone id (bus.zone)                             */
  const int32_t* load_bus;    /* [n_load]                                               */
  const double* load_scaling; /* [n_load]                                   [1]         */
  const int32_t* sgen_bus;    /* [n_sgen]                                               */
  const int32_t* sgen_zone;   /* [n_sgen] zone id (sgen.name)                           */
  const double* sgen_scaling; /* [n_sgen]                                   [1]         */
} mapdn_net_desc;

/*
 * Profile store - the three CSVs after pv_scale / demand_scale (replaces reference
 * _load_pv_data/_load_active_demand_data/_load_reactive_demand_data :407-438). HOST arrays,
 * row-major [n_rows, n], copied to HBM once. std/s_max as the reference derives them in
 * __init__ (:70-73, :515-521).
 */
typedef struct {
  int64_t n_rows;
  int32_t steps_per_hour;     /* 60 // time_delta (reference :389,396)                  */
  int32_t n_days;             /* (index[-1] - index[0]).days (reference :395)           */
  const double* pv;           /* [n_rows, n_sgen] MW                                    */
  const double* load_p;       /* [n_rows, n_load] MW                                    */
  const double* load_q;       /* [n_rows, n_load] MVAr                                  */
  const double* pv_std;       /* [n_sgen]  data.std(axis=0)/100                         */
  const double* load_p_std;   /* [n_load]                                               */
  const double* load_q_std;   /* [n_load]                                               */
  const double* s_max;        /* [n_sgen]  1.2 * max_t pv                               */
} mapdn_profile_desc;

/* env_args (reference args/env_args/var_voltage_control.yaml:3-20, read at :46-84) */
typedef struct {
  int32_t batch;              /* number of independent env instances on this device     */
  int32_t barrier;            /* mapdn_barrier                                          */
  double voltage_weight;      /* [1.0]                                                  */
  double q_weight;            /* [0.1]; ignored when use_line_weight                    */
  double line_weight;
  int32_t use_line_weight;    /* line_weight != None (reference :612)                   */
  double v_upper, v_lower;    /* [1.05, 0.95]                                           */
  int32_t episode_limit;      /* [240]                                                  */
  double action_low, action_high; /* action_bias -/+ action_scale (reference :76)       */
  int32_t reset_action;       /* random initial q at reset (reference :120-122)         */
  uint64_t seed;              /* Philox key                                             */
  int64_t env_id_offset;      /* global id of env 0 (multi-GPU shards; RNG is keyed by  */
                              /* global env id so results do not depend on the sharding)*/
  double tol;                 /* NR tolerance on ||F||inf p.u. [1e-8]; <=0 => default   */
  int32_t max_iter;           /* NR iteration cap [10]; <=0 => default                  */
  int32_t lanes_per_env;      /* 0 = auto; else 4, 8, 16, 32, 64 or 128 threads per env */
  int32_t state_space_mask;   /* state_space (reference :78): bit0 demand, bit1 pv, bit2 reactive, bit3 vm_pu,
                                 bit4 va_degree; 0 = all five (the default)              */
} mapdn_cfg;

typedef struct {
  int32_t batch, n_bus, n_branch, n_line, n_load, n_sgen;
  int32_t n_agents, n_actions, obs_dim, state_dim, n_info;
  int32_t lanes_per_env, envs_per_block, smem_bytes, n_levels;
  int64_t algorithmic_bytes_per_env_step; /* SURVEY §8d formula                         */
} mapdn_dims;

typedef struct mapdn_env mapdn_env;

int32_t mapdn_abi_version(void);
const char* mapdn_last_error(void);

/* replaces VoltageControl.__init__ (reference :36-94) minus file parsing */
mapdn_status mapdn_create(const mapdn_net_desc* net, const mapdn_profile_desc* prof,
                          const mapdn_cfg* cfg, int32_t device, mapdn_env** out);
mapdn_status mapdn_destroy(mapdn_env* env);
mapdn_status mapdn_get_dims(const mapdn_env* env, mapdn_dims* out);

/*
 * reset / manual_reset (reference :96-176). start_dhi_dev: int32 [B,3] = (day, hour, interval)
 * per env (manual_reset semantics) or NULL to sample hour/day/interval on the device
 * (reference :381-398). Envs whose initial power flow diverges are re-drawn on the device
 * (reference retry loop :108-133; the reference retries for ever, the device gives up after 16
 * draws per call and reports it: converged_dev [B] uint8, 1 = solved, 0 = every draw diverged -
 * call again with those envs in mask_dev). mask_dev: uint8 [B] (NULL = all) selects envs to
 * reset; converged_dev is written for the selected envs only. A manual start outside the
 * profile store is clamped to the last window that fits. Outputs may be NULL.
 */
mapdn_status mapdn_reset(mapdn_env* env, const int32_t* start_dhi_dev, const uint8_t* mask_dev,
                         int32_t add_noise, double* obs_dev /*[B,n_agents,obs_dim]*/,
                         double* state_dev /*[B,state_dim]*/, uint8_t* converged_dev /*[B] or NULL*/,
                         void* stream);

/*
 * step (reference :178-211): q = a*sqrt(s_max^2 - p_pv^2) -> Newton-Raphson power flow ->
 * reward / info (or the divergence branch) -> next profile row (+|N(0,1)|*std noise) ->
 * steps += 1 -> terminated. obs_dev (optional) receives get_obs() of the new state (:232-316).
 * One fused kernel launch.
 */
mapdn_status mapdn_step(mapdn_env* env, const double* actions_dev /*[B,n_sgen]*/, int32_t add_noise,
                        double* reward_dev /*[B]*/, uint8_t* terminated_dev /*[B]*/,
                        double* info_dev /*[B,11] or NULL*/, double* obs_dev /*or NULL*/,
                        void* stream);

/* Same through HOST buffers: H2D of actions, kernel, D2H of the results, stream sync. */
mapdn_status mapdn_step_host(mapdn_env* env, const double* actions_host, int32_t add_noise,
                             double* reward_host, uint8_t* terminated_host, double* info_host,
                             double* obs_host, void* stream);

/*
 * Host path without staging copies: every buffer must be page-locked host memory (cudaHostAlloc / cudaHostRegister;
 * unified addressing). The fused kernel reads the actions from and writes reward / terminated / info / observations
 * to host memory directly, so the PCIe transfer of the observations overlaps the kernel instead of following it.
 * obs_is_f32: obs_host is float [B,n_agents,obs_dim] instead of double. skip_padding: the zero padding at the end of
 * each agent's row (reference :270-274; it never changes) is not rewritten - the caller zero-fills obs_host once.
 * sync = 0 returns right after the launch (results are valid after mapdn_wait / a stream synchronisation): the
 * caller's policy for the next step can run while the device works.
 */
mapdn_status mapdn_step_host_pinned(mapdn_env* env, const double* actions_host, int32_t add_noise,
                                    double* reward_host, uint8_t* terminated_host, double* info_host,
                                    void* obs_host, int32_t obs_is_f32, int32_t skip_padding, int32_t sync,
                                    void* stream);
mapdn_status mapdn_wait(mapdn_env* env, void* stream);

/*
 * Host path with compact observation rows. get_obs (reference :232-316) pads every agent's row with zeros up to the
 * longest one (:270-274); here the host receives obs_host [B, row_len] (double, or float when obs_is_f32) in which agent a
 * owns entries [agent_off[a], agent_off[a] + agent_len[a]) - its reference row without the padding (row_len = sum of
 * the lengths, rounded up to a multiple of 4 with zeros). The kernel writes the compact rows into device memory and ONE
 * contiguous copy-engine transfer moves them (long contiguous rows are what the copy engine moves fastest); actions are read from and reward / terminated / info written to host memory directly. All
 * host buffers must be page-locked. direct = 1: the kernel writes the compact rows to obs_host itself instead (no
 * device staging, no copy; on an H100 about as fast end to end as the copy). sync as in
 * mapdn_step_host_pinned.
 */
mapdn_status mapdn_obs_compact_layout(const mapdn_env* env, int32_t* agent_off /*[n_agents]*/,
                                      int32_t* agent_len /*[n_agents]*/, int32_t* row_len);
mapdn_status mapdn_step_host_compact(mapdn_env* env, const double* actions_host, int32_t add_noise,
                                     double* reward_host, uint8_t* terminated_host, double* info_host,
                                     void* obs_host, int32_t obs_is_f32, int32_t direct, int32_t sync,
                                     void* stream);

/*
 * Variants that deliver the observations in fp32 - what the reference's learners consume (prep_obs casts to
 * float32 right away, reference utilities/util.py:137-147). Halves the device->host traffic of the host-buffer
 * path; everything else (reward, info, the env state itself) stays fp64.
 */
mapdn_status mapdn_step_f32obs(mapdn_env* env, const double* actions_dev, int32_t add_noise, double* reward_dev,
                               uint8_t* terminated_dev, double* info_dev, float* obs_dev, void* stream);
mapdn_status mapdn_step_host_f32obs(mapdn_env* env, const double* actions_host, int32_t add_noise,
                                    double* reward_host, uint8_t* terminated_host, double* info_host,
                                    float* obs_host, void* stream);

/*
 * Tester records (reference utilities/tester.py:26-55): after manual_reset and after every step the tester reads six
 * getters. A record row holds them side by side, fp64, in the tester's key order:
 *   [pv_active n_sgen | pv_reactive n_sgen | bus_active n_bus | bus_reactive n_bus | bus_voltage n_bus | line_loss n_line]
 * = the values mapdn_get_field returns for P_SGEN, Q_SGEN, P_BUS, Q_BUS, VM, LINE_LOSS at that moment (after a step
 * pv_active is already the next profile row, as in the reference; a diverged step reports the previous results).
 * mapdn_record_layout: off[MAPDN_N_RECORD] = start of each of the six blocks, row_len = entries per row.
 * mapdn_record: one gather launch writing the current row of env b to record_dev + b * record_stride (stride in
 * doubles, >= row_len) - after a reset.
 * mapdn_step_record: mapdn_step (same arguments, same outputs) whose kernel also writes every env's row after the step
 * from the values it already holds - no extra launch. record_dev = NULL is exactly mapdn_step.
 */
#define MAPDN_N_RECORD 6
mapdn_status mapdn_record_layout(const mapdn_env* env, int32_t* off /*[MAPDN_N_RECORD]*/, int32_t* row_len);
mapdn_status mapdn_record(mapdn_env* env, double* record_dev, int64_t record_stride, void* stream);
mapdn_status mapdn_step_record(mapdn_env* env, const double* actions_dev /*[B,n_sgen]*/, int32_t add_noise,
                               double* reward_dev /*[B]*/, uint8_t* terminated_dev /*[B]*/,
                               double* info_dev /*[B,11] or NULL*/, double* obs_dev /*or NULL*/,
                               double* record_dev /*or NULL*/, int64_t record_stride, void* stream);

/*
 * Observation history (env_args `history`, reference :87, :303-315): with history = H > 1 every get_obs() returns each
 * agent's last H frames side by side, oldest first, zero frames before the episode start - rows [n_agents, H*obs_dim].
 * mapdn_set_history(H): H > 1 allocates a zero-filled frame ring on the device [B, H, n_agents*obs_dim]; from then on
 * every reset and every step (any mapdn_step* entry point, obs requested or not) records the env's newest frame in it.
 * Frame f of an env counts the frames since its last reset (the reset gives f = 0) and lives in slot f mod H, so a reset
 * clears nothing. H = 1 frees the ring; H < 1 is refused.
 * mapdn_step_stacked: mapdn_step_record (same arguments, same outputs) whose kernel also writes the stacked rows
 * [B, n_agents, H*obs_dim] to obs_stacked_dev (may be NULL) - one launch.
 * mapdn_get_obs_stacked: one gather launch writing the same rows from the ring (after a reset or a host-path step).
 * Both refuse a handle without history. mapdn_dims.obs_dim stays the width of one frame.
 */
mapdn_status mapdn_set_history(mapdn_env* env, int32_t history);
mapdn_status mapdn_step_stacked(mapdn_env* env, const double* actions_dev /*[B,n_sgen]*/, int32_t add_noise,
                                double* reward_dev /*[B]*/, uint8_t* terminated_dev /*[B]*/,
                                double* info_dev /*[B,11] or NULL*/, double* obs_dev /*or NULL*/,
                                double* obs_stacked_dev /*[B,n_agents,H*obs_dim] or NULL*/,
                                double* record_dev /*or NULL*/, int64_t record_stride, void* stream);
mapdn_status mapdn_get_obs_stacked(mapdn_env* env, double* obs_stacked_dev, void* stream);

/*
 * Step with auto-reset: an env that terminates in the step (steps >= episode_limit or a diverged power flow) starts its
 * next episode in the same launch. One launch whose results equal, call for call, those of
 *   1. mapdn_step (obs_stacked_dev NULL) / mapdn_step_stacked with the same arguments (no records);
 *   2. mapdn_reset(env, NULL, mask = terminated_dev, add_noise = 1, obs = reset_obs_dev, state = NULL,
 *      converged = reset_ok_dev): sampled start, noise on, up to the reset's own number of draws; an env whose draws
 *      all diverge keeps its power-flow results (res_*) and, like any reset env, starts the new episode's counters
 *      (steps = 1, sum_rewards, start_row, episode) with the element values of its last draw;
 *   3. with history, mapdn_get_obs_stacked into reset_obs_stacked_dev, for the terminated envs.
 * obs_dev / obs_stacked_dev keep the step's (terminal) observation; reset_obs_dev [B,n_agents,obs_dim],
 * reset_obs_stacked_dev [B,n_agents,H*obs_dim] and reset_ok_dev [B] are written for the terminated envs only (each may
 * be NULL). Refuses a null handle, actions, reward or terminated, a handle without a profile store, and stacked
 * pointers on a handle without history.
 */
mapdn_status mapdn_step_autoreset(mapdn_env* env, const double* actions_dev /*[B,n_sgen]*/, int32_t add_noise,
                                  double* reward_dev /*[B]*/, uint8_t* terminated_dev /*[B]*/,
                                  double* info_dev /*[B,11] or NULL*/, double* obs_dev /*or NULL*/,
                                  double* obs_stacked_dev /*or NULL*/, double* reset_obs_dev /*or NULL*/,
                                  double* reset_obs_stacked_dev /*or NULL*/, uint8_t* reset_ok_dev /*or NULL*/,
                                  void* stream);

/*
 * Env state snapshots: save the state of any envs of the batch into device memory and put it back, into the same or
 * other slots, of this handle or of another one with the same layout.
 * A snapshot row holds one env's whole state, bytes_per_env bytes (a multiple of 16): one segment per state array, in the
 * order of the list below, each starting 16-byte aligned, zero padding behind it. HIST is the observation history's
 * frame ring [H, n_agents*obs_dim], empty when history = 1. Element types: fp64, except START_ROW int64, STEPS and
 * NR_ITERS int32, EPISODE uint32.
 * mapdn_snapshot_layout: off[s] = byte offset of segment s in a row, off[MAPDN_N_SNAPSHOT] = bytes_per_env. The layout
 * depends on the net and on the handle's current history (mapdn_set_history): a row can only be restored into a handle
 * whose layout is the same.
 * mapdn_snapshot: row k of buf_dev (at buf_dev + k * bytes_per_env) receives the state of env idx_dev[k];
 * mapdn_restore: env idx_dev[k] receives row k. idx_dev: int32 [n] on the device, or NULL for all envs in order (then n
 * must equal the batch). Entries outside [0, batch) are skipped (nothing read or written for them). Duplicate entries in
 * a restore list are a caller error: the result is undefined. buf_dev must be 16-byte aligned. One launch each,
 * stream-ordered, no host synchronisation. Both refuse a null handle or buffer, n <= 0, n > batch, idx_dev = NULL with
 * n != batch and a handle without a profile store.
 * Noise. The Philox streams of the noise are keyed by the seed, the global env id (env_id_offset + slot), the episode
 * counter and the step. The counter and the step are state; the seed and the global id are not. So restoring an env's
 * own row into a slot with the same global id (on any handle with the same seed, in any process) replays its future bit
 * for bit under the same actions. A row restored into a slot with another global id (a fork) draws that slot's noise:
 * the first step after the fork still gives the source's reward, info and power flow (its profile row was drawn before
 * the snapshot), the rows drawn after differ unless add_noise = 0.
 */
#define MAPDN_N_SNAPSHOT 15   /* segments: CUR_PL, CUR_QL, CUR_PV, CUR_Q, RES_VM, RES_VA, RES_P, RES_Q, RES_PL,
                                 SUM_REWARDS, START_ROW, STEPS, EPISODE, NR_ITERS, HIST (empty when history = 1) */
mapdn_status mapdn_snapshot_layout(const mapdn_env* env, int64_t* off /*[MAPDN_N_SNAPSHOT + 1]; last = bytes_per_env*/);
mapdn_status mapdn_snapshot(mapdn_env* env, const int32_t* idx_dev /*[n] or NULL*/, int32_t n, void* buf_dev,
                            void* stream);
mapdn_status mapdn_restore(mapdn_env* env, const int32_t* idx_dev /*[n] or NULL*/, int32_t n, const void* buf_dev,
                           void* stream);

mapdn_status mapdn_get_obs(mapdn_env* env, double* obs_dev, void* stream);      /* :232-316 */
mapdn_status mapdn_get_state(mapdn_env* env, double* state_dev, void* stream);  /* :213-230 */
mapdn_status mapdn_get_field(mapdn_env* env, int32_t field, double* out_dev, void* stream);

/*
 * Stateless batched power flow = pp.runpp on explicit element values (parity / benchmark
 * entry; reference call sites :124,:165,:557). nb envs (any nb >= 1; independent of cfg.batch).
 * Inputs dev fp64: p_load,q_load [nb,n_load], p_sgen,q_sgen [nb,n_sgen]. Outputs (each may be
 * NULL): vm, va_deg [nb,n_bus]; p_bus,q_bus [nb,n_bus] (res_bus.p_mw/q_mvar); pl [nb,n_line];
 * iters int32 [nb]; converged uint8 [nb].
 */
mapdn_status mapdn_solve(mapdn_env* env, int32_t nb, const double* p_load, const double* q_load,
                         const double* p_sgen, const double* q_sgen, double* vm, double* va_deg,
                         double* p_bus, double* q_bus, double* pl, int32_t* iters,
                         uint8_t* converged, void* stream);

/*
 * Droop-control baseline of the paper, one control instant per env in ONE launch (reference
 * traditional_control/pf_droop_matpower_all.m:121-152 loop, :196-231 q(v) characteristic): starting from q = 0, run
 * the power flow, stop when ||v_pv - v_pv_prev||_2 < tol, else q <- (1 - gain) q + gain q_droop(v_pv); at most max_ite
 * power flows (script: gain 0.1, tol 1e-4, max_ite 100). Inputs dev fp64: p_load,q_load [nb,n_load], p_sgen [nb,n_sgen],
 * s_rated, q_max_manual [n_sgen]. Outputs: vm [nb,n_bus] (may be NULL), q_sgen [nb,n_sgen] = the q of the last power
 * flow, loss [nb] = sum of res_line.pl_mw, iterations int32 [nb] = power flows run. No host synchronisation.
 */
mapdn_status mapdn_droop(mapdn_env* env, int32_t nb, const double* p_load, const double* q_load,
                         const double* p_sgen, const double* s_rated, const double* q_max_manual,
                         double gain, double tol, int32_t max_ite, double* vm, double* q_sgen,
                         double* loss, int32_t* iterations, void* stream);

/* Ybus as assembled on the device (dense row-major complex [n_bus,n_bus] -> two host arrays);
 * test hook for the makeYbus restatement. */
mapdn_status mapdn_get_ybus_dense(mapdn_env* env, double* g_host, double* b_host);

/* Number of kernels of this library launched since the handle was created. */
int64_t mapdn_launch_count(const mapdn_env* env);

#ifdef __cplusplus
}
#endif
#endif /* MAPDN_B200_H */
