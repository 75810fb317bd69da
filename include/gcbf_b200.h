/*
 * gcbf_b200.h -- C ABI of libgcbf_b200.so: the sm_90a (H100) hot path of GCBF+
 * (batched rollout step + GCBF+ train step) behind plain pointers and sizes.
 *
 * The reference (MIT-REALM/gcbfplus) has NO FFI / plugin / operator layer: its hot
 * path is XLA code generated from Python (SURVEY.md 1, 8b).  Each entry point
 * below therefore names the reference *Python* function(s) it replaces
 * (paths relative to the reference root); INTEGRATION.md shows the ctypes
 * binding a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in _host;
 *   - the caller owns all memory (inputs, outputs, workspace); the library never
 *     allocates, frees or retains device memory across calls;
 *   - all calls are asynchronous on `stream` (a cudaStream_t passed as void*),
 *     re-entrant, and CUDA-graph capturable (no host sync, no allocation);
 *   - return value: 0 = ok; < 0 = argument / configuration error, nothing was
 *     enqueued; > 0 = cudaError_t of a failed launch.  gcbf_last_error_string()
 *     describes the last non-zero return of the calling thread;
 *   - fp32 everywhere, int32 indices, uint8 masks.
 *
 * Batch layout ("swarm batch", SURVEY 8a1): G graphs x N agents, A = G*N.
 *   agent  [G,N,sd]   goal [G,N,sd]   hits [G,N,R,pd]  (pd = 2 or 3)
 *   obstacles: Rectangle [G,O,16] = cx,cy,w/2,h/2,cos,sin,p0x,p0y,...,p3x,p3y,0,0
 *              Sphere    [G,O,4]  = cx,cy,cz,radius
 *   edges (receiver-grouped lists, replaces utils/graph.py:35-44,209-244):
 *     row_start[A], row_deg[A]; edge_recv[e] = global agent id of the receiver;
 *     edge_src[e]  >= 0  : global agent id of the sending agent
 *                  == -1 : the receiver's own goal node
 *                  <= -2 : the receiver's hit node k = -2 - edge_src[e]
 *     per receiver the order is [goal | agents ascending j | active hits ascending k].
 */
#ifndef GCBF_B200_H
#define GCBF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GCBF_ENV_SINGLE_INTEGRATOR 0
#define GCBF_ENV_DOUBLE_INTEGRATOR 1
#define GCBF_ENV_DUBINS_CAR 2
#define GCBF_ENV_LINEAR_DRONE 3

#define GCBF_NET_CBF 0
#define GCBF_NET_ACTOR 1

#define GCBF_MSG_HID 256
#define GCBF_MSG_DIM 128

/* Environment / batch descriptor.  Python-float constants of the reference are
 * rounded to fp32 by the HOST exactly where JAX's weak typing rounds them (e.g.
 * lidar_radius = float32(comm_radius - 1e-1)). */
typedef struct gcbf_env_desc {
    int32_t env_kind;       /* GCBF_ENV_* */
    int32_t n_graphs;       /* G */
    int32_t n_agents;       /* N */
    int32_t n_obs;          /* O obstacles per graph (0 allowed) */
    int32_t n_rays;         /* rays cast per agent (2-D: n_rays <= 32; 3-D: (n/2)*n+2) */
    int32_t n_hits;         /* R hit nodes kept per agent */
    int32_t edge_cap;       /* capacity of edge_recv / edge_src and of per-edge workspaces */
    int32_t obs_per_graph;  /* 1: obstacles [G,O,..]; 0: one obstacle set shared by all graphs */
    float comm_radius;      /* params["comm_radius"] */
    float comm_radius_p1;   /* comm_radius + 1 (self-edge removal, double_integrator.py:230) */
    float lidar_radius;     /* comm_radius - 1e-1 (double_integrator.py:257) */
    float dt;               /* env/__init__.py:44 */
    float mass;             /* DoubleIntegrator params["m"] */
    float radius;           /* car_radius / drone_radius */
    float two_r;            /* radius * 2 */
    float two_r_p1;         /* radius * 2 + 1 */
    float half_r;           /* radius * 0.5 (Dubins stop mask) */
    float unsafe_agent;     /* agent-agent unsafe distance (2r; LinearDrone 2.5r) */
    float unsafe_obs;       /* obstacle inflation in unsafe_mask (r; Dubins/LD 1.5r) */
    float warn_agent;       /* 3r */
    float warn_obs;         /* 2r */
    float four_r_sq;        /* 4 * r**2 */
    float r_sq;             /* r**2 */
    float safe_agent;       /* safe_mask distance (4r; SI 2.5r) */
    float safe_obs;         /* safe_mask inflation (2r; SI 1.5r) */
    float comm_sq_thr;      /* smallest fp32 a with sqrtf(a) >= comm_radius:  (sqrtf(x) < Rc) == (x < comm_sq_thr) */
    float lidar_sq_thr;     /* same for lidar_radius */
    float v_lim;            /* state_lim on velocity components (inf if none) */
    float u_lim;            /* action_lim */
    float K[18];            /* LQR gain [nu, sd] row-major (u_ref), fp32 */
    float A[36];            /* LinearDrone A [sd,sd] row-major (continuous), fp32 */
    float B[18];            /* LinearDrone B [sd,nu] row-major, fp32 */
} gcbf_env_desc;

/* ---------------------------------------------------------------- misc */
const char* gcbf_last_error_string(void);
int32_t gcbf_version(void);
/* number of thread-block launches of this library's kernels since process start
 * (host-side counter; used by bench.py for "gpu_launches"). */
int64_t gcbf_launch_count(void);
/* size in floats of the flat parameter buffer of a network with n_layers GNN layers (gnn.py:78-104;
 * 1 <= n_layers <= 8) and its offset table: W,b of the 9 Dense layers of GNN layer 0, ..., of layer n_layers - 1, then
 * of the 3 head layers (2 * (9 * n_layers + 3) entries, forward order, see DESIGN.md; n_layers = 1: 24 entries, the
 * reference's 12 Dense layers).  From layer 1 on, msg/Dense_0 is [ed + 256, 256] and update/Dense_0 is [256, 256]. */
int32_t gcbf_param_count_l(int32_t edge_dim, int32_t out_dim, int32_t n_layers);
int32_t gcbf_param_offsets_l(int32_t edge_dim, int32_t out_dim, int32_t n_layers, int32_t* offsets_host);

/* ---------------------------------------------------------------- graph build (a1,a2,a3)
 * Replaces env.get_graph: get_lidar/raytracing/inside_obstacles
 * (gcbfplus/env/utils.py:49-131, env/obstacle.py:53-96,234-270) and edge_blocks +
 * GetGraph.to_padded (env/double_integrator.py:223-264,288-320;
 * utils/graph.py:35-44,209-244) for G graphs at once.
 * flags bit0: 1 = cast rays and write `hits`; 0 = `hits` is an input (topology only).
 * counters[0] <- number of edges; counters[1] |= 1 on edge_cap overflow (sticky).
 * Canonical layout: rows in batch-agent order, row_start[0] = 0, row_start[a + 1] = row_start[a] + row_deg[a],
 * counters[0] = sum of row_deg; every output is bit-identical from run to run (row contents after an overflow are
 * unspecified).  flags bit3: keep the rows where the build placed them (ticket order, one launch fewer than the
 * canonical pass) -- for callers whose results do not depend on the layout, such as rollouts. */
int32_t gcbf_graph_build(const gcbf_env_desc* desc, const float* agent, const float* obstacles,
                         const float* ray_table, float* hits, int32_t* row_start, int32_t* row_deg,
                         int32_t* edge_recv, int32_t* edge_src, int32_t* counters, int32_t flags,
                         void* stream);

/* ---------------------------------------------------------------- GNN forward (a4,a5)
 * Replaces CBF.get_cbf / DeterministicPolicy.get_action: GNNLayer + head MLP + tanh
 * (gcbfplus/nn/gnn.py:44-104, nn/mlp.py:6-30, algo/module/cbf.py:12-53,
 * algo/module/policy.py:63-128), including env.add_edge_feats when clip_all = 1
 * (env/double_integrator.py:275-286).
 * params: flat fp32 buffer of n_layers GNN layers (gcbf_param_offsets_l).  out: [A, out_dim] (tanh applied).
 * params_t: NULL -> strict-fp32 SIMT GEMMs (n_layers = 1 only); else the tf32 hi / lo planes of the GEMM weights from
 * gcbf_prepare_params_l (gcbf_params_t_count_l floats) -> wgmma tensor-core GEMMs (3xTF32 split, fp32 accumulate;
 * same tolerance).  From layer 1 on, S = y Ws and R = y Wr are node-level GEMMs and each edge gathers
 * S[sender] + R[receiver]; goal and hit nodes, which never receive a message, are one constant row each per layer.
 * workspace: gcbf_gnn_workspace_floats_l() floats; at n_layers = 1 it holds the saved activations the backward pass
 * reads. */
int64_t gcbf_gnn_workspace_floats_l(const gcbf_env_desc* desc, int32_t out_dim, int32_t n_layers);
int32_t gcbf_params_t_count_l(int32_t edge_dim, int32_t out_dim, int32_t n_layers);
int32_t gcbf_prepare_params_l(int32_t edge_dim, int32_t out_dim, int32_t n_layers, const float* params,
                              float* params_t, void* stream);
int32_t gcbf_gnn_forward_l(const gcbf_env_desc* desc, int32_t net_kind, int32_t out_dim, int32_t n_layers,
                           const float* params, const float* params_t, const float* agent, const float* goal,
                           const float* hits, const int32_t* row_start, const int32_t* row_deg,
                           const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
                           int32_t clip_all, float* out, float* workspace, int64_t workspace_floats, void* stream);

/* Inference-only forward with FOLDED weights (rollouts; same functions replaced as gcbf_gnn_forward_l).
 * Each MLP block ends in two activation-free linear layers (nn/mlp.py:23-29, act_final=False), which are
 * multiplied together once per parameter update by gcbf_prepare_infer: 4 GEMMs instead of 9 per forward and
 * 2.4x fewer FLOPs; no activations are saved.  infer_blob: gcbf_infer_count() floats (folded weights, their
 * transposed and straight tf32 hi / lo planes, U2 U3 for the train step's un-folding). */
int32_t gcbf_infer_count(int32_t edge_dim, int32_t out_dim);
int32_t gcbf_prepare_infer(int32_t edge_dim, int32_t out_dim, const float* params, float* infer_blob,
                           void* stream);
int32_t gcbf_gnn_infer(const gcbf_env_desc* desc, int32_t net_kind, int32_t out_dim, const float* params,
                       const float* infer_blob, int32_t use_tensor_cores, const float* agent,
                       const float* goal, const float* hits, const int32_t* row_start,
                       const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src,
                       const int32_t* counters, int32_t clip_all, float* out, float* workspace,
                       int64_t workspace_floats, void* stream);

/* ---------------------------------------------------------------- env step (a6,a7)
 * Replaces GCBFPlus.act/step (algo/gcbf_plus.py:176-186: a = 2 pi + u_ref) and
 * env.step minus get_graph (env/double_integrator.py:145-198: clip_action,
 * agent_step_euler, reward, get_cost).
 * mode 0: action <- 2*pi + u_ref (output);  mode 1: `action` is an INPUT (env.step(graph, action));
 * mode 2: action <- u_ref (test.py --u-ref);  mode 3: as mode 1 with the DubinsCar stop mask off
 * (env.enable_stop = False, env/dubins_car.py:138-142, which DecShareCBF sets; other envs: same as mode 1).
 * Outputs: action [A,nu] (unclipped a, what the rollout records), next_agent [A,sd],
 * reward [G], cost [G]. */
int32_t gcbf_env_step(const gcbf_env_desc* desc, const float* agent, const float* goal,
                      const float* obstacles, const float* pi, const int32_t* row_start,
                      const int32_t* row_deg, const int32_t* edge_src, float* action,
                      float* next_agent, float* reward, float* cost, int32_t mode, void* stream);
/* action [A,nu] <- (pi ? 2*pi : 0) + u_ref(agent, goal): GCBFPlus.act (algo/gcbf_plus.py:176-180)
 * and env.u_ref (env/double_integrator.py:332-338, env/dubins_car.py:328-379). */
int32_t gcbf_act(const gcbf_env_desc* desc, const float* agent, const float* goal, const float* pi,
                 float* action, void* stream);

/* ---------------------------------------------------------------- reset (f3)
 * Start / goal positions of every environment: get_node_goal_rng (gcbfplus/env/utils.py:134-226) with
 * jax.random's threefry key chain, one warp per environment.
 *   keys [G, 2] uint32 (device): the key get_node_goal_rng receives (after the obstacle draws of env.reset,
 *     env/double_integrator.py:89-104); obstacles: packed, one set per environment
 *   area_size, min_dist (= 4 * radius), max_travel (< 0: none)
 *   agent / goal [G, N, sd] (device): the position components are written, the rest is left untouched. */
int32_t gcbf_reset_positions(const gcbf_env_desc* desc, const uint32_t* keys, const float* obstacles,
                             float area_size, float min_dist, float max_travel, float* agent, float* goal,
                             void* stream);
/* Same with the threefry stream layout selectable: threefry_partitionable = 0 -> jax's legacy layout (default of
 * the 0.4.x line, what gcbf_reset_positions uses); 1 -> jax_threefry_partitionable=True (default from JAX 0.5.0:
 * split child i = threefry(key, (0, i)), random bits = y0 ^ y1).  The reference does not pin a JAX version
 * (requirements.txt: jax>=0.4.14), so "identical seeds" is defined per layout. */
int32_t gcbf_reset_positions_ex(const gcbf_env_desc* desc, const uint32_t* keys, const float* obstacles,
                                float area_size, float min_dist, float max_travel, int32_t threefry_partitionable,
                                float* agent, float* goal, void* stream);

/* ---------------------------------------------------------------- fused rollout step (a8 body)
 * One iteration of the scan body of rollout() (gcbfplus/trainer/utils.py:46-49): algo.step
 * (algo/gcbf_plus.py:182-186) + env.step incl. get_graph of the next state
 * (env/double_integrator.py:145-181) for the G envs of the batch, 5 kernel launches and no
 * memset / copy in between: policy forward with folded weights (4 launches: edge features + message
 * layer with the gate layer chained onto the tile -> logits, segment softmax + aggregate, update
 * layer, folded update/head layer with the output layer's partial sums in its epilogue) -> one
 * kernel that applies the policy tail
 * {tanh head, a = 2 pi + u_ref, clip, Euler} for the whole graph in every CTA, records actions /
 * next states / per-env reward and cost, and builds LiDAR hits + neighbour lists of the next state.
 * The NEXT graph (next_row_start ... next_counters) must not alias the current one: callers
 * double-buffer the edge lists (the cost of the step reads the current lists while the next ones are
 * written).  counters / next_counters are the 4-int counter blocks of the current / next graph.
 * n_layers > 1 (tensor-core path only): infer_blob is the gcbf_prepare_params_l output instead of the
 * gcbf_prepare_infer one, the policy forward runs layer by layer unfolded (gcbf_gnn_forward_l) and the same policy
 * tail + graph build kernel ends the step.
 * workspace: gcbf_rollout_workspace_floats_l(). */
int64_t gcbf_rollout_workspace_floats_l(const gcbf_env_desc* desc, int32_t n_layers);
int32_t gcbf_rollout_step_l(const gcbf_env_desc* desc, int32_t n_layers, const float* actor_params,
                            const float* infer_blob, int32_t use_tensor_cores, const float* agent,
                            const float* goal, const float* obstacles, const float* ray_table, const float* hits,
                            const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
                            const int32_t* edge_src, const int32_t* counters, float* action, float* next_agent,
                            float* next_hits, int32_t* next_row_start, int32_t* next_row_deg,
                            int32_t* next_edge_recv, int32_t* next_edge_src, int32_t* next_counters,
                            float* reward, float* cost, float* workspace, int64_t workspace_floats,
                            void* stream);

/* Measurement hook: the same step with only the launches whose bit is set in `select` enqueued (bench.py times every
 * kernel of the step alone, on the buffers a full step left behind, to find the dominant one and its roofline):
 * bit 0 edge features + message layer + chained gate layer, bit 1 segment softmax + aggregate, bit 2 update layer,
 * bit 3 folded update/head layer, bit 4 policy tail + graph build of the next state.  GCBF_STEP_ALL = the whole step
 * (gcbf_rollout_step_l at n_layers = 1; workspace: gcbf_rollout_workspace_floats_l(desc, 1)). */
#define GCBF_STEP_ALL 31
int32_t gcbf_rollout_step_select(const gcbf_env_desc* desc, const float* actor_params, const float* infer_blob,
                                 int32_t use_tensor_cores, const float* agent, const float* goal,
                                 const float* obstacles, const float* ray_table, const float* hits,
                                 const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
                                 const int32_t* edge_src, const int32_t* counters, float* action,
                                 float* next_agent, float* next_hits, int32_t* next_row_start,
                                 int32_t* next_row_deg, int32_t* next_edge_recv, int32_t* next_edge_src,
                                 int32_t* next_counters, float* reward, float* cost, float* workspace,
                                 int64_t workspace_floats, int32_t select, void* stream);

/* ---------------------------------------------------------------- persistent rollout (a8 whole scan)
 * The WHOLE rollout() of gcbfplus/trainer/utils.py:25-55 (reset excluded) in ONE kernel launch: one thread-block cluster
 * per environment loops over the n_steps env-steps; the kernel boundaries of gcbf_rollout_step_l become cluster barriers,
 * pipeline / table setup is paid once per rollout (csrc/rollout_persist.cu).  Same arithmetic as
 * gcbf_rollout_step_l -> same bits.  Supported: SingleIntegrator / DoubleIntegrator / DubinsCar, n_agents <= 512,
 * n_obs <= 32, one obstacle set per environment, desc->edge_cap >= n_graphs * n_agents (it is split evenly over the
 * environments); gcbf_rollout_persistent_supported() tells, callers fall back to gcbf_rollout_step_l otherwise.
 *   agent_rec [n_steps+1, G, N, sd]: slice 0 = initial states (input), slices 1.. written;  hits_rec [n_steps+1, G, N, R, pd]
 *   (all slices written, slice 0 = LiDAR of the initial states);  actions_rec [n_steps, G, N, nu];  rewards / costs
 *   [n_steps, G];  counters [n_steps+1, 4] (zeroed by the caller): [t][0] += edges of the graphs of state t, [t][1] |= overflow.
 *   workspace: gcbf_rollout_persistent_workspace_floats(desc) floats, 256-byte aligned.
 *   phase_stamps: NULL, or [(n_steps + 1) * 8 + 2 * G] uint64 (device): first [n_steps + 1][8]: %globaltimer (ns) of environment 0's first CTA at the phase
 *   boundaries of every step (start, after edge phase, aggregate, update GEMM, head GEMM, policy tail, LiDAR + neighbour
 *   bits, end) -- the in-kernel profile bench.py reports (row 0 = the initial graph build); then [G][2] = start / end time
 *   of every environment's cluster (shows whether all clusters were co-resident). */
int64_t gcbf_rollout_persistent_workspace_floats(const gcbf_env_desc* desc);
/* 0: unsupported; 1: supported but the environments' clusters are not all co-resident on this device (environments
 * beyond the resident clusters wait for a free slot and the rollout takes two rounds); 2: supported and
 * co-resident (the case callers should pick it for). */
int32_t gcbf_rollout_persistent_supported(const gcbf_env_desc* desc);
/* co-resident clusters of `cluster_size` CTAs of the persistent kernel on the current device (occupancy query) */
int32_t gcbf_rollout_persistent_max_clusters(int32_t cluster_size);
int32_t gcbf_rollout_persistent(const gcbf_env_desc* desc, int32_t n_steps, const float* actor_params,
                                const float* infer_blob, const float* goal, const float* obstacles,
                                const float* ray_table, float* agent_rec, float* hits_rec, float* actions_rec,
                                float* rewards, float* costs, int32_t* counters, float* workspace,
                                int64_t workspace_floats, uint64_t* phase_stamps, void* stream);
/* The persistent rollout of several one-layer actors in ONE launch: environment g runs network net_of_env[g].  Each
 * cluster reads its network once, at its start, and runs the operations of gcbf_rollout_persistent in the same order, so
 * every network's environments get the bits a gcbf_rollout_persistent launch of that network alone gives them (the
 * environments never read one another's data).
 *   actor_params [n_nets, param_stride]: network k's flat parameters (gcbf_param_count_l(ed, nu, 1) floats) at
 *   k * param_stride;  infer_blob [n_nets, infer_stride]: network k's gcbf_prepare_infer output (gcbf_infer_count(ed, nu)
 *   floats) at k * infer_stride.  The strides are those counts rounded up to a multiple of 4 floats (16 bytes: the
 *   stride of the 3-D weight tensor maps, network outermost); gcbf_rollout_persistent_multi_strides returns them.  Both
 *   arrays 16-byte aligned.
 *   net_of_env [G] int32 (device): every entry in [0, n_nets).  The library does not read it on the host; an entry out
 *   of range is the caller's bug (undefined reads).
 *   counters [n_steps+1, n_nets, 4] (zeroed by the caller): [t][k][0] += edges of the graphs of state t of network k's
 *   environments, [t][k][1] |= their overflow.  Every other argument as gcbf_rollout_persistent (desc->n_graphs = G
 *   counts the environments of all networks; workspace: gcbf_rollout_persistent_workspace_floats(desc)).
 * Unlike gcbf_rollout_persistent it also launches when gcbf_rollout_persistent_supported(desc) is 1 and the pair mode
 * does not fit the device: the clusters beyond the resident ones then run in later rounds (none waits on another).
 * Rejected before anything is enqueued: n_nets < 1, a NULL net_of_env, misaligned stacked arrays, and whatever
 * gcbf_rollout_persistent rejects. */
int32_t gcbf_rollout_persistent_multi(const gcbf_env_desc* desc, int32_t n_steps, int32_t n_nets,
                                      const float* actor_params, const float* infer_blob, const int32_t* net_of_env,
                                      const float* goal, const float* obstacles, const float* ray_table,
                                      float* agent_rec, float* hits_rec, float* actions_rec, float* rewards,
                                      float* costs, int32_t* counters, float* workspace, int64_t workspace_floats,
                                      uint64_t* phase_stamps, void* stream);
/* Per-network strides (floats) of gcbf_rollout_persistent_multi's stacked actor_params / infer_blob for edge_dim /
 * out_dim (one GNN layer).  0, or -1 for bad dimensions. */
int32_t gcbf_rollout_persistent_multi_strides(int32_t edge_dim, int32_t out_dim, int64_t* param_stride,
                                              int64_t* infer_stride);

/* ---------------------------------------------------------------- labels / masks (a9)
 * Replaces env.unsafe_mask / collision_mask / finish_mask / safe_mask
 * (env/double_integrator.py:356-440 and twins).  Any output pointer may be NULL.
 * Outputs uint8 [A]. */
int32_t gcbf_masks(const gcbf_env_desc* desc, const float* agent, const float* goal,
                   const float* hits, const float* obstacles, uint8_t* unsafe, uint8_t* collision,
                   uint8_t* finish, uint8_t* safe, void* stream);
/* GCBFPlus.safe_mask horizon labelling (algo/gcbf_plus.py:160-174).
 * unsafe/safe: uint8 [n_rollouts, T, N]. */
int32_t gcbf_safe_horizon(const uint8_t* unsafe, uint8_t* safe, int32_t n_rollouts, int32_t T,
                          int32_t n_agents, int32_t horizon, void* stream);

/* ---------------------------------------------------------------- train step (a10, a11)
 * gcbf_train_step replaces one `update_fn` of GCBFPlus.update_inner up to (not including) the
 * optimizer (gcbfplus/algo/gcbf_plus.py:356-434): h = cbf(g); a = 2 pi(g) + u_ref; g' =
 * env.forward_graph(g, a); h' = cbf(g'); loss = c_a mean||a - u_qp||^2 + c_u unsafe + c_s safe +
 * c_h mean relu(-h_dot - alpha h + eps) with the reference's stop-gradient routing for
 * unlabelled agents (:399-407); jax.value_and_grad wrt (cbf_params, actor_params).
 *   hp_host[7] (HOST): alpha, eps, loss_action_coef, loss_unsafe_coef, loss_safe_coef, loss_h_dot_coef,
 *     use_tensor_cores (0: strict-fp32 SIMT GEMMs, layer by layer; 1: wgmma 3xTF32 GEMMs on the FOLDED network --
 *     the activation-free layer pairs of every MLP block multiplied together as in gcbf_prepare_infer, the
 *     gradient un-folded onto the flax parameters by the chain rule; same gradient, ~1e-6 relative rounding)
 *   denoms[4] (device): GLOBAL n_unsafe, n_safe, n_agents of the minibatch (gcbf_mask_counts, then
 *     summed over ranks by the host when the minibatch is sharded)
 *   grad_cbf / grad_actor: flat gradients in the parameter layout (overwritten)
 *   stats[16] (device, overwritten): LOCAL numerators 0 sum relu(h+eps)[unsafe], 1 sum relu(-h+eps)[safe],
 *     2 sum relu(-h_dot-alpha h+eps), 3 sum ||a-u_qp||^2, 4 #(h<0 & unsafe), 5 #(h>0 & safe),
 *     6 #(h_dot+alpha h>0), 7 n_unsafe, 8 n_safe, 9 n_agents
 *   workspace: gcbf_train_workspace_floats(desc) floats.
 * Deterministic: no float atomics -- every sum over CTAs is taken in a fixed order (per-CTA partials, then an ordered
 * sum; per-edge input gradients gathered per agent) -- so grad_cbf, grad_actor and stats are bit-identical from run to
 * run for the same inputs and edge layout on the same GPU model (the SM count sets the split counts).
 * Sharded training: ranks call this on their shard with the global denoms, then sum
 * [grad_cbf | grad_actor | stats] with ONE all-reduce before gcbf_clip_adamw. */
int64_t gcbf_train_workspace_floats(const gcbf_env_desc* desc);
int32_t gcbf_mask_counts(const uint8_t* safe_mask, const uint8_t* unsafe_mask, int32_t n_agents_total,
                         float* denoms, void* stream);
int32_t gcbf_train_step(const gcbf_env_desc* desc, const float* hp_host, const float* cbf_params,
                        const float* actor_params, const float* agent, const float* goal,
                        const float* hits, const int32_t* row_start, const int32_t* row_deg,
                        const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
                        const uint8_t* safe_mask, const uint8_t* unsafe_mask, const float* u_qp,
                        const float* denoms, float* grad_cbf, float* grad_actor, float* stats,
                        float* workspace, int64_t workspace_floats, void* stream);
/* out[0] = sum g^2, out[1] = number of non-finite entries (trainer/utils.py:62-64 compute_norm);
 * out must hold 2 + 512 floats (out[2..] = scratch partials).  Deterministic (no float atomics) so
 * that every rank derives the same clip scale from the all-reduced gradient. */
int32_t gcbf_grad_sqnorm(const float* grad, int32_t n, float* out, void* stream);
/* compute_norm_and_clip (trainer/utils.py:66-75) + optax.adamw(lr, b1, b2, eps, weight_decay) wrapped in
 * optax.apply_if_finite (gcbf_plus.py:109-110,127-128): g <- g / max(max_norm, ||g||) * max_norm; if any
 * gradient entry is non-finite nothing is changed; step[0] (device int32) counts applied updates. */
int32_t gcbf_clip_adamw(float* params, const float* grad, float* m, float* v, int32_t n,
                        const float* norm_info, int32_t* step, float lr, float b1, float b2, float eps,
                        float weight_decay, float max_norm, void* stream);
/* tgt <- tau * src + (1 - tau) * tgt  (GCBFPlus.update_tgt, gcbf_plus.py:188-191). */
int32_t gcbf_polyak(float* tgt, const float* src, int32_t n, float tau, void* stream);

/* ---------------------------------------------------------------- QP action labels (f1)
 * gcbf_qp_labels replaces GCBFPlus.get_b_u_qp / get_qp_action (gcbfplus/algo/gcbf_plus.py:193-196,
 * 299-352; the JaxProxQP solve at :341-346) for a batch of graphs: per graph
 *   min_{u,r} 1/2|u|^2 - u_ref.u + 5|r|^2 + 1000 sum(r)
 *   s.t.  -Lg_h u - r <= Lf_h + 0.1 alpha h,   -u_lim <= u <= u_lim,   r >= 0
 * with h = cbf(add_edge_feats(graph, x)) (all edge features norm-clipped), h_x its Jacobian wrt the
 * agent states (one data-only backward pass kept per edge: h is a one-layer GNN, so row i touches
 * only agent i and its neighbours), f, g = env.control_affine_dyn.  Solved exactly (unique
 * minimiser) by an accelerated projected-gradient ascent on the dual, one CTA per graph.
 *   cbf_params: the parameters to label with (the reference passes the TARGET network, :210)
 *   max_iter / tol: iteration cap and stopping threshold on the projected dual-gradient residual
 *   u_qp [G, N, nu] (out);  aux [G, N, 2] = (multiplier lam, relaxation r) or NULL;  iters [G] or NULL
 *     (iteration count; bit 30 set when the graph was too dense for the shared-memory path)
 *   workspace: gcbf_qp_workspace_floats(desc) floats;  n_agents <= 2048.
 * gcbf_qp_workspace_layout: float offsets inside the workspace of the assembled QP (test hook):
 *   0 h[A]  1 JE[cap,8] (d h_recv / d feat_e)  2 b[A]  3 Lg_self[A,4]  4 Lg_edge[cap,4]  5 u_ref[A,4]
 *   6 row scale[A]  7 mirror-edge index[cap] (int32). */
int64_t gcbf_qp_workspace_floats(const gcbf_env_desc* desc);
int32_t gcbf_qp_workspace_layout(const gcbf_env_desc* desc, int64_t* offsets8_host);
int32_t gcbf_qp_labels(const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores, int32_t max_iter,
                       float tol, const float* cbf_params, const float* agent, const float* goal,
                       const float* hits, const int32_t* row_start, const int32_t* row_deg,
                       const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
                       float* u_qp, float* aux, int32_t* iters, float* workspace, int64_t workspace_floats,
                       void* stream);
/* gcbf_qp_filter: the learned-CBF safety filter.  The QP of gcbf_qp_labels with a nominal action in place of u_ref:
 *   min_{u,r} 1/2|u|^2 - u_nom.u + 5|r|^2 + 1000 sum(r)   (same constraints)
 * i.e. the action closest to u_nom that keeps the CBF condition (relaxed by r where no admissible action does).
 *   u_nom [G, N, nu]: the nominal action (the policy's 2 pi + u_ref, or any other); may lie outside the u_lim box.
 *     NULL: u_ref, and then every output is bit-identical to gcbf_qp_labels'.
 *   u [G, N, nu] (out), aux, iters, workspace (gcbf_qp_workspace_floats) and the other arguments as gcbf_qp_labels.
 * The solve's sums run over the edge lists in row order, so the result depends on the layout: callers that need
 * deterministic results pass canonical graphs (gcbf_graph_build without flags bit3). */
int32_t gcbf_qp_filter(const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores, int32_t max_iter,
                       float tol, const float* cbf_params, const float* agent, const float* goal,
                       const float* hits, const int32_t* row_start, const int32_t* row_deg,
                       const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
                       const float* u_nom, float* u, float* aux, int32_t* iters, float* workspace,
                       int64_t workspace_floats, void* stream);

/* ---------------------------------------------------------------- online policy refinement
 * gcbf_refine_actions replaces GCBF.online_policy_refinement (gcbfplus/algo/gcbf.py:161-201, inherited by GCBFPlus)
 * for a batch of G graphs, each with its own stopping rule:
 *   h = cbf(g);  v_ref = relu(-(cbf(forward_graph(g, u_ref)) - h) / dt - alpha h)   (per agent)
 *   a = where(v_ref > 0, 2 pi + u_ref, u_ref);  i = 0, val = 1
 *   while val > 0 and i < max_iter:  val = mean_agents relu(-(cbf(forward_graph(g, a)) - h) / dt - alpha h),
 *                                    a -= lr * d val / d a,  i += 1
 * (the reference's constants: lr = 0.1, max_iter = 30).  The gradient runs through clip_action, the Euler step,
 * clip_state and the recomputed edge features with the train step's conventions (relu'(0) = 0, zero gradient outside
 * the clip limits, the DubinsCar stop mask).  The launch sequence is fixed (capturable in a CUDA graph, no host sync);
 * once every graph has stopped the remaining iterations run with zero device row counts.  One-layer CBF only.
 *   cbf_params / cbf_prepared: the CBF parameters and gcbf_refine_prepare's planes of them (rebuild them whenever
 *     the parameters change): the tf32 planes (use_tensor_cores != 0) or the transposed weights of the strict-fp32
 *     SIMT path;
 *     gcbf_params_t_count_l(edge_dim, 1, 1) floats
 *   pi [A, nu]: the actor output (policy.get_action);  graph arrays as gcbf_qp_labels takes them
 *   action [A, nu] (out): the refined actions;  value [G] or NULL: the last loop value of each graph
 *   iters [G] or NULL: iterations taken, bit 30 set when the graph stopped at max_iter with value > 0
 *   workspace: gcbf_refine_workspace_floats(desc) floats.
 * Deterministic: the same inputs on the same GPU model give bit-identical action, value and iters. */
int32_t gcbf_refine_prepare(int32_t edge_dim, int32_t use_tensor_cores, const float* cbf_params, float* prepared,
                            void* stream);
int64_t gcbf_refine_workspace_floats(const gcbf_env_desc* desc);
int32_t gcbf_refine_actions(const gcbf_env_desc* desc, float alpha, float lr, int32_t max_iter,
                            int32_t use_tensor_cores, const float* cbf_params, const float* cbf_prepared,
                            const float* pi, const float* agent, const float* goal, const float* hits,
                            const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
                            const int32_t* edge_src, const int32_t* counters, float* action, float* value,
                            int32_t* iters, float* workspace, int64_t workspace_floats, void* stream);

/* ---------------------------------------------------------------- CBF-QP baseline controllers
 * Replace the reference's hand-written baselines for a batch of G graphs: the pairwise CBFs
 * (gcbfplus/algo/utils.py:44-349, get_pwise_cbf_fn :413-439, k = 3), DecShareCBF.get_qp_action
 * (algo/dec_share_cbf.py:61-150) and CentralizedCBF.get_qp_action (algo/centralized_cbf.py:64-117).
 * Candidates of agent i: [the N agents of its graph | its own R hit nodes], squared distance with the self entry at
 * 100, the 3 nearest in stable order.  Inputs: agent / goal [G,N,sd], hits [G,N,R,pd].
 *
 * gcbf_cbf_pairwise (get_cbf + the Lie terms of its jax.jacfwd):
 *   k_idx [G,N,3] int32: candidate index (j < N: agent j of the graph; N + k: hit node k of this agent);
 *   k_isobs [G,N,3] uint8 (k_idx >= N);  k_h, k_lf_h [G,N,3];  k_lg_self [G,N,3,nu] = dh/dx_i g(x_i);
 *   k_lg_other [G,N,3,nu] = dh/dx_j g(x_j) for an agent pick j != i, else 0 (NULL: not written).
 *   k_lf_h includes the picked agent's drift: dh/dx_i f(x_i) + dh/dx_j f(x_j).
 * gcbf_cbfqp_dec_share: one QP per agent, x = [u (nu) | r (3)],
 *   min 1/2|u|^2 - u_ref.u + 5|r|^2 + 1000 sum r  s.t.  -Lg_self u - r <= resp (Lf_h + alpha h),  |u| <= u_lim,  r >= 0,
 *   resp = 1 for an obstacle pick, 0.5 for an agent pick.  u [G,N,nu]; r [G,N,3] or NULL;
 *   iters [G,N] or NULL (solves: one per agent).
 * gcbf_cbfqp_centralized: one QP per graph, x = [u (N nu) | r (3N)], rows (i, k) with Lg blocks of agent i and of
 *   the picked agent, b = Lf_h + alpha h.  n_agents <= GCBF_CBFQP_CENTRAL_MAX_AGENTS, LinearDrone <= 999 (the
 *   graph's QP lives in shared memory; larger is rejected with status -1).  u [G,N,nu]; r [G,N,3] or NULL; iters [G] or NULL (solves: one per graph).
 * Both solve the dual exactly in fp64 (unique minimiser): max_iter caps the iterations, tol is the stopping threshold
 * on the projected dual-gradient residual.  iters[s] = iterations of solve s, with bit 30 set when the cap was hit
 * before the stopping test passed (the iterate at the cap is returned).
 *   workspace: gcbf_cbfqp_workspace_floats(desc) floats (holds the pairwise terms). */
#define GCBF_CBFQP_CENTRAL_MAX_AGENTS 1024
int32_t gcbf_cbf_pairwise(const gcbf_env_desc* desc, const float* agent, const float* hits, int32_t* k_idx,
                          uint8_t* k_isobs, float* k_h, float* k_lf_h, float* k_lg_self, float* k_lg_other,
                          void* stream);
int64_t gcbf_cbfqp_workspace_floats(const gcbf_env_desc* desc);
int32_t gcbf_cbfqp_dec_share(const gcbf_env_desc* desc, float alpha, int32_t max_iter, float tol, const float* agent,
                             const float* goal, const float* hits, float* u, float* r, int32_t* iters,
                             float* workspace, int64_t workspace_floats, void* stream);
int32_t gcbf_cbfqp_centralized(const gcbf_env_desc* desc, float alpha, int32_t max_iter, float tol,
                               const float* agent, const float* goal, const float* hits, float* u, float* r,
                               int32_t* iters, float* workspace, int64_t workspace_floats, void* stream);

/* ---------------------------------------------------------------- dense-layer building blocks
 * The fp32 GEMM family the MLPs are made of (flax nn.Dense, gcbfplus/nn/mlp.py:19-21, and its
 * autodiff transposes).  Exported so the kernels can be unit-tested against a plain fp32
 * reference and timed in isolation by bench.py; row-major contiguous operands.
 * gemm_nn: C[M,N] = epi(A[M,K] @ B[K,N]);  epi 0: +bias(+bias2), 1: relu(+bias(+bias2)),
 *          2: none, 3: aux > 0 ? acc : 0;  accum != 0: C += (epi 2/3 only).
 *          M = *m_ptr (device) if m_ptr else m_fixed, clamped to m_cap.  K % 16 == 0, N % 128 == 0.
 * gemm_tn: C[K1,N] += sum_m w(m) X[m, :K1] dY[m, :N]  (ldx = row stride of X; w optional:
 *          roww[row2agent ? row2agent[m] : m]).  K1, N multiples of 128.
 * colsum : db[N] += sum_m w(m) dY[m, :N], N in {128, 256}. */
int32_t gcbf_gemm_nn(int32_t epi, int32_t accum, const float* A, const float* B, const float* bias,
                     const float* bias2, float* C, const float* aux, const int32_t* m_ptr,
                     int32_t m_fixed, int32_t m_cap, int32_t K, int32_t N, void* stream);
/* gemm_tc: the wgmma tensor-core variant (3xTF32 split, fp32 accumulation in registers, TMA-staged
 * operands): C[M,N] = epi(A[M,K] @ Bt[N,K]^T) with Bt = the TRANSPOSED weight (K-major operands);
 * Bt is passed as its tf32 split Bt_hi + Bt_lo (gcbf_split_tf32; weights are split once per update);
 * same epilogues / row-count convention as gemm_nn, plus EPI_RELU_DOTN = 5
 * (C[(part * m_cap + m) * 4 + q] = relu(acc + bias) . aux[:, q] over the 128 columns of column tile `part`,
 * q < ndot <= 4, the other q written 0); epi = 4 is not an epilogue and returns an error.
 * K % 32 == 0, N in {128, 256}; A must be backed by at least m_cap rows. */
int32_t gcbf_gemm_tc(int32_t epi, int32_t accum, const float* A, const float* Bt_hi, const float* Bt_lo,
                     const float* bias, const float* bias2, float* C, const float* aux,
                     const int32_t* m_ptr, int32_t m_fixed, int32_t m_cap, int32_t K, int32_t N, int32_t ndot,
                     void* stream);
/* hi = tf32(x) (round to nearest), lo = tf32(x - hi): the operand split of the 3xTF32 scheme. */
int32_t gcbf_split_tf32(const float* in, float* hi, float* lo, int32_t n, void* stream);
int32_t gcbf_gemm_tn(const float* X, int32_t ldx, const float* dY, float* C, const float* roww,
                     const int32_t* row2agent, const int32_t* m_ptr, int32_t m_fixed, int32_t m_cap,
                     int32_t K1, int32_t N, int32_t n_agents_total, void* stream);
/* gemm_tn_tc: wgmma variant of gemm_tn (operands transposed to K-major in shared memory, 3xTF32 split, split-M + red.add);
 * cs1 / cs2 (optional): += sum_m w(m) dY[m, :N], the column sums taken from the same pass over dY. */
int32_t gcbf_gemm_tn_tc(const float* X, int32_t ldx, const float* dY, float* C, const float* roww,
                        const int32_t* row2agent, const int32_t* m_ptr, int32_t m_fixed, int32_t m_cap,
                        int32_t K1, int32_t N, int32_t n_agents_total, float* cs1, float* cs2,
                        void* stream);
int32_t gcbf_colsum(const float* dY, float* db, const float* roww, const int32_t* row2agent,
                    const int32_t* m_ptr, int32_t m_fixed, int32_t m_cap, int32_t N,
                    int32_t n_agents_total, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GCBF_B200_H */
