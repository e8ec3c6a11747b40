// Kernel-side view of one mapdn_env handle: pointers into HBM + scalars, passed by value.
#pragma once
#include <stdint.h>

namespace mapdn {

// Per-env shared memory: (npq + 2) node records of 9 double2 (144 B, array-of-structs: one address
// computation per node, 128-bit accesses; the bank group of field f of node i is (i + f) mod 8, so node ids that differ
// mod 8 never conflict - mapdn_create picks the ids accordingly), then the sgen block (pv | q), then a scratch region:
// [n_sgen] next pv row / droop voltages, the partials of the multi-warp reductions, and the staged loads unless they are
// staged inside the records (DESIGN.md section 2).
// Record npq is a sentinel: the slack bus in VV / EF / SP, all-zero in UP / DN / T / R (the "no child" /
// "no parent" slot of the branch-free gathers). Record npq + 1 is a trash record: idle lanes of a
// schedule step work on it so that the level sweeps have no divergent branches.
constexpr int kNodeArrays2 = 9;
enum NodeArr2 {           // index of the double2 field inside a node record
  A_VV = 0,   // (|V|, theta)
  A_EF,       // (e, f) = V in rectangular form
  A_SP,       // (P_spec, Q_spec) p.u. injections (Sbus); slack slot: computed injection (P0, Q0)
  A_UP,       // (a, b) of J[i, parent]      -> after elimination: S01 (first row of the Schur update)
  A_DN,       // (a, b) of J[parent, i]      -> after elimination: S23
  A_T,        // J[parent,i] D^-1 r  (rhs update for the parent)
  A_D01,      // diagonal block row 0        -> after elimination: M01 = (D^-1 J[i,parent]) row 0
  A_D23,      // diagonal block row 1        -> after elimination: M23
  A_R         // rhs (-F)                    -> D^-1 r -> dx
};
// epilogue aliases (the Newton arrays are dead by then)
constexpr int A_BP = A_D01;   // res_bus (p_mw, q_mvar) per node
constexpr int A_OP = A_D23;   // "demand" columns of get_obs: res_bus p/q + sgen add-back (reference :238-244)
constexpr uint32_t kNone = 0xFFFFu;   // "no parent" in 16-bit node fields
// esched flags: low 8 bits = number of children beyond two; then where child 0's Schur update comes from
constexpr unsigned kEschedReg0 = 0x100u;    // registers of the same lane (it eliminated child 0 in the previous step)
constexpr unsigned kEschedLoad0 = 0x200u;   // shared memory
constexpr unsigned kEschedLoad1 = 0x400u;   // child 1 exists (always from shared memory)
constexpr unsigned kEschedIdle = 0x1000u;   // idle lane of this step: reads the trash record, stores nothing
constexpr unsigned kEschedLeaf = 0x2000u;   // no child at all: the update is zero (no shared-memory access on the step's chain)
constexpr unsigned kEschedStore = 0x800u;   // the parent will read this bus's Schur update from shared memory
// bsched flags (bits 32.. of an entry)
constexpr unsigned kBschedRegParent = 0x1u; // dx of the parent is in this lane's registers (it solved the parent in the previous step)
constexpr unsigned kBschedIdle = 0x2u;      // idle lane of this step (trash record)

struct HotLayout {        // byte offsets inside the hot static blob (staged into smem per CTA)
  int yup, ydn;           // double2 [npq], [npq + 1]: Y[i,parent], Y[parent,i]   (G, B); ydn[npq] = 0 ("no child")
  int yii;                // double2 [npq]: Y[i,i]
  int tables_in_blob;     // the four once-per-step tables below are part of the blob (else: the cold copies in Params)
  int ysl;                // double2 [npq]: Y[i,slack]
  int obs_off;            // uint16 [n_sgen*obs_dim]: obs entry -> double offset inside the env slab
  int line_nodes;         // uint16 [2*n_line]: from / to node of every line (npq = slack)
  int line_c;             // double [4*n_line]: loss coefficients (see mapdn_b200.cu)
  int ndesc;              // uint64 [npq]: node descriptor, see below
  int esched;             // uint64 [n_esteps * G]: elimination schedule, one entry per (step, lane):
                          //   node | child0<<16 | child1<<32 | flags<<48   (idle lane: trash record)
  int bsched;             // uint64 [n_bsteps * G]: back-substitution schedule: node | parent<<16 | kBsched* flags<<32
                          //   (levels 1.. of the forest: the roots' dx = D^-1 r is already in place)
  int lptr, lidx;         // uint16 [npq+2], [n_load]: node -> loads (CSR); node npq = slack bus
  int sptr, sidx;         // uint16 [npq+2], [n_sgen]: node -> sgens
  int xptr, xidx;         // uint16 [npq+2], [<=n_sgen]: node -> sgens of the node's own zone (obs add-back)
  int node_of_bus;        // uint16 [n_bus]: bus -> node (slack -> npq)
  int nbr_ptr, nbr_idx;   // meshed nets only: uint16 CSR of the PQ-PQ Ybus pattern ([npq+1], [nnz])
  int nbr_y;              // meshed nets only: double2 [nnz]: Y[i,j] (G, B) of each CSR entry
  int bytes;              // total, multiple of 16
};

// node descriptor (64 bit):
//   bits  0-15 parent (the sentinel record npq for roots: zero admittance)
//   bits 16-31 first child  (npq = none -> zero slot)
//   bits 32-47 second child (npq = none)
//   bits 48-62 number of children beyond two (they follow child1 contiguously)
//   bit  63    the bus is adjacent to the slack bus (Y[i,slack] in the cold table ysl)
struct Params {
  // ---- sizes ----
  int n_bus, npq, n_load, n_sgen, n_line, n_lev, obs_dim, state_dim, n_slack_adj, slack_bus;
  int n_esteps, n_bsteps, has_extra_children;   // schedule lengths (for the handle's G); any bus with > 2 children
  int n_wide_e, n_narrow_b;                     // G > 32: forward steps >= n_wide_e and back steps < n_narrow_b occupy lanes 0..31 only
  int nb;                 // envs processed by this launch
  int helper_threads;     // MODE_STEP: threads of the helper warps behind the solver threads of a CTA
  int env_stride2;        // double2 elements of smem per env
  int pvq_off2;           // double2 offset of the sgen (pv | q) block inside the env slab
  int scratch_off2;       // double2 offset of the scratch region (prologue staging / next-row prefetch)
  int stage_in_records;   // the prologue stages the scaled loads in the (dead) Newton fields of the node records
  int helper_off;         // byte offset (in the CTA's dynamic smem) of the helper warps' per-env scalars: int4 [envs per CTA]
  int has_shunt;          // any bus shunt: res_bus p/q get the shunt power (cold tables sh_g / sh_b)
  HotLayout hot_layout;
  const unsigned char* hot;
  // ---- cold static (global, read through the read-only path) ----
  const int* bus_of_node;                                     // [npq]
  const double* lscale; const double* sscale;                 // scaling by load id / sgen id
  const int* sl_node; const double* sl_y;                     // slack-adjacent nodes, Y[slack,i] (G,B)
  // cold copies of the once-per-step tables (used when they are left out of the shared-memory blob: large nets)
  const double2* ysl;                                         // [npq] Y[i,slack] (zero unless adjacent to the slack)
  const uint16_t* obs_off;                                    // [n_sgen*obs_dim] obs entry -> double offset in the env slab
  const uint16_t* line_nodes;                                 // [2*n_line] from / to node of every line (npq = slack)
  const double* line_c;                                       // [4*n_line] loss coefficients (see mapdn_b200.cu)
  const int* sgen_node;                                       // [n_sgen] node of each sgen's bus (slack -> npq)
  // the static first Newton iteration (flat start): per node S_calc, M rows 0/1, D'^-1 rows 0/1, J[parent,i]
  const double2* first_tab;                                   // [6 * npq]
  const double* sh_g; const double* sh_b;                     // [npq + 1] bus shunt GS / BS (MW / MVAr at 1 p.u.) by node
  const unsigned* obs_src; const int* obs_xptr; const int* obs_xidx;   // cold obs program of get_obs_kernel
  const unsigned* state_src;                                  // state program: kind | bus / sgen index
  const double* s_max; const double* pv_std; const double* lp_std; const double* lq_std;
  // ---- profile store ----
  const double* prof_pv; const double* prof_lp; const double* prof_lq;
  long long n_rows; int steps_per_hour; int n_day_choices;
  // ---- scalars ----
  double base_mva, inv_base, vm_init, e0, f0, vm0, va0, ysl_g0, ysl_b0, tol;   // ysl_*0 = Y[slack,slack]
  int max_iter;
  int barrier; double voltage_weight, q_weight, line_weight; int use_line_weight;
  double v_upper, v_lower; int episode_limit; double action_low, action_high; int reset_action;
  unsigned long long seed; long long env_id_offset;
  // ---- env state (global, [B, *]) ----
  double* cur_pl; double* cur_ql; double* cur_pv; double* cur_q;
  double* res_vm; double* res_va; double* res_p; double* res_q; double* res_pl;
  int* steps; double* sum_rewards; long long* start_row; unsigned* episode;
  int* nr_iters;          // Newton iterations of the env's last power flow (max_iter when it diverged)
  // ---- launch io ----
  const double* in_pl; const double* in_ql; const double* in_pv; const double* in_q;  // SOLVE
  const double* actions;                                                             // STEP
  const int* start_dhi; const unsigned char* mask; int add_noise;                    // RESET
  unsigned char* reset_ok;                                                           // RESET: [B] 1 = the env's power flow converged
  double* out_vm; double* out_va; double* out_p; double* out_q; double* out_pl;
  int* out_iters; unsigned char* out_conv;
  // DROOP (traditional_control/pf_droop_matpower_all.m): rated S and manual q limit per sgen, relaxation, outputs
  const double* droop_s; const double* droop_qmm; double droop_gain, droop_tol; int droop_max_ite;
  double* droop_q_out; double* droop_loss_out;
  double* reward; unsigned char* term; double* info; double* obs; double* state;
  float* obs32;           // alternative fp32 destination of the observations (MODE_STEP)
  int obs_skip_off;       // slab offset whose obs entries are NOT stored: -1 (store everything) or the zero slot (host
                          // path into a buffer whose padding is already zero: a third fewer bytes over PCIe)
  const uint16_t* obs_compact_prog;  // the same program without the per-agent zero padding (rows of obs_compact_len entries)
  int obs_compact_len;    // > 0: observations are written as compact rows (mapdn_step_host_compact); 0: padded layout
  double* dense_ws;       // meshed nets only: per resident env group, (2 npq) x (2 npq + 1) doubles [J | rhs]
  int dense_stride;       // doubles per group in dense_ws
  long long* prof;        // MAPDN_PROFILE builds: per-phase clock64 totals of warp 0 of block 0
  // tester records (mapdn_step_record / mapdn_record): row of env b at record + b * record_stride (doubles), laid out
  // [pv n_sgen | q n_sgen | P_bus n_bus | Q_bus n_bus | vm n_bus | line loss n_line]
  double* record;
  long long record_stride;
  // observation history (mapdn_set_history, history > 1): frame ring [B][history][n_sgen * obs_dim] (the padded get_obs
  // layout). Frame f of an env counts the frames since its last reset (f = steps - 1) and lives in slot f mod history.
  double* hist;
  int history;            // 1: no ring
  // MODE_STEP of a handle with history (or NULL): stacked rows [B, n_sgen, history * obs_dim], oldest frame first, zero
  // frames before the episode start (reference get_obs :303-315)
  double* obs_stacked;
  // auto-reset step (mapdn_step_autoreset, or NULL): first observation of the new episode of every env that terminated in
  // the step ([B, n_sgen, obs_dim]) and, with history, its stacked row ([B, n_sgen, history * obs_dim]); reset_ok above
  // takes the reset outcome
  double* reset_obs;
  double* reset_obs_stacked;
};

// cold obs program entry: kind in the top 4 bits, node / sgen index in the low 28
enum ObsKind { OBS_ZERO = 0, OBS_P = 1, OBS_Q = 2, OBS_PV = 3, OBS_QSG = 4, OBS_VM = 5, OBS_VA = 6,
               OBS_PBUS = 7, OBS_QBUS = 8, OBS_VA_DEG = 9 };   // the last three: get_state (bus index, no add-back)

}  // namespace mapdn
