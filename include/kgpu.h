/*
 * kgpu.h -- C ABI of libkgpu: the H100-native topology-aware GPU placement scorer
 * that replaces the scoring path of microsoft/KubeGPU's gpuschedulerplugin.
 *
 * This is the drop-in boundary (SURVEY.md 8(b)).  A Go host binds these entry
 * points through cgo (`#include "kgpu.h"`, see INTEGRATION.md); in this
 * repository they are exercised through ctypes (kubegpu_b200/_lib.py) and through
 * the C++ host mirror of the reference's DeviceScheduler interface
 * (kubegpu_b200/csrc/host/).  Plain pointers and sizes only -- no C++/torch types.
 *
 * What each group replaces in the reference (/root/reference, commit 73e59ce):
 *   kgpu_upload_nodes / kgpu_update_node / kgpu_remove_node
 *       <- NvidiaGPUScheduler.AddNode / RemoveNode   gpuschedulerplugin/gpu_scheduler.go:21-32
 *          (node cache: AddResourcesToNodeTreeCache   gpuschedulerplugin/gpu.go:192-230);
 *          the matrix is the one nvml.GetDevices builds nvidiagpuplugin/gpu/nvml/nvml.go:37-49
 *   kgpu_score_batch[_device]
 *       <- NvidiaGPUScheduler.PodFitsDevice (score)   gpuschedulerplugin/gpu_scheduler.go:34-44
 *          -> TranslatePodGPUResources                gpuschedulerplugin/gpu.go:94-127
 *          -> findBestTreeInCache + assignGPUs        gpuschedulerplugin/gpu.go:232-271
 *          batched over every (pod, node) pair instead of one cgo call per pair
 *   kgpu_fit_lookup / kgpu_build_fit_table / kgpu_score_pairs
 *       <- the same PodFitsDevice, called once per (node, pod) by the core: served from a host-side (node, k) table
 *   kgpu_set_free_mask[s] / kgpu_place_batch[_ex|_gang|_gang_domain|_gang_levels] / kgpu_upload_domain[s|_levels] /
 *   kgpu_get_free_masks
 *       <- TakePodResources / ReturnPodResources       gpuschedulerplugin/gpu_scheduler.go:57-63 (no-ops there)
 *   kgpu_reduce_shards_device
 *       <- (no reference counterpart; the reference is single-process) the final
 *          per-pod pick over the all-gathered shard results, SURVEY.md 8(e)
 *   kgpu_set_weights
 *       <- the link-level grouping tables {6,5,4} / {6,5,4,3,2,1}
 *          nvidiagpuplugin/gpu/nvidia/nvidia_gpu_manager.go:178-180
 *   kgpu_last_error
 *       <- Go `error` returns (gpu_scheduler.go:46-55, gpu.go:125-126)
 *
 * Data layouts (all little-endian, host or device as stated per function):
 *   topo       int32[N][64]   row-major 8x8 link-level matrix per node; only the
 *                             upper triangle (i<j) is read; values 0..15
 *                             (0 unknown, 1..6 NVML P2P level, 7..12 NVLink links).
 *   free_mask  int32[N]       bit i = GPU i present and free (low 8 bits).
 *   pods       int32[P][4]    {k, pod_id, flags, min_mem_mib}; k GPUs wanted, 0..8;
 *                             min_mem_mib > 0: only GPUs with at least that much memory are
 *                             eligible for this pod (see kgpu_upload_gpu_memory); pod_id/flags
 *                             are carried, not interpreted.
 *   gpu_mem    int32[N][8]    MiB per GPU slot (the node agent advertises it per GPU as
 *                             `.../memory`, nvidia_gpu_manager.go:204-211); optional.
 *   keys       uint64[P]      (cost << 40) | (node_id << 8) | gpu_mask, or
 *                             KGPU_NO_FIT.  cost = sum over GPU pairs i<j in the
 *                             mask of W[topo[i][j]]; the key is the minimum over
 *                             all nodes and all k-subsets of free GPUs, so ties go
 *                             to the lower node_id, then the lower mask.
 *
 * Threading: every call on one handle is serialised by an internal mutex.  State-changing calls (upload, update,
 * set_free_mask(s), place_batch) and the lazy rebuilds they trigger run on the handle's own stream and have COMPLETED
 * when the call returns, so a following launch on any stream sees them.  The *_device entry points only enqueue: all
 * such calls on one handle must go to ONE stream at a time (the handle's per-batch scratch -- the "batch has
 * memory-constrained pods" flag, the work list -- is not duplicated per stream); use one handle per stream otherwise.
 * Errors: functions return KGPU_OK (0) or a negative KGPU_ERR_*; the message is
 * kept per handle (kgpu_last_error(h)) and per thread (kgpu_last_error(NULL)).
 * "No node fits" is a result (KGPU_NO_FIT), never an error.  Nothing here falls
 * back to the CPU: without a usable CUDA device every call fails.
 */
#ifndef KGPU_H_
#define KGPU_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGPU_OK 0
#define KGPU_ERR_INVALID (-1) /* bad argument / value out of domain          */
#define KGPU_ERR_CUDA (-2)    /* CUDA runtime error (message has the detail) */
#define KGPU_ERR_NOMEM (-3)   /* host or device allocation failed            */
#define KGPU_ERR_COMM (-4)    /* NCCL / peer-access failure (multi-device)   */
#define KGPU_ERR_STATE (-5)   /* call not valid in the handle's state        */

#define KGPU_NO_FIT UINT64_MAX
#define KGPU_MAX_GPUS_PER_NODE 8
#define KGPU_NUM_LEVELS 16
#define KGPU_MAX_WEIGHT 4095

/* Kernel variants of K1 `score_pairs` (all bit-identical in result). */
#define KGPU_VARIANT_AUTO 0          /* default: the cheapest path with identical keys for the batch at hand: pods without a
                                      * memory requirement are memoised by k (best[k] over all nodes once, then a gather),
                                      * pods with one are scored per pair by the memory-aware kernel (K1m)          */
#define KGPU_VARIANT_WARP_PER_PAIR 1 /* north_star mapping: warp per (pod,node), lane per subset */
#define KGPU_VARIANT_LANE_PER_NODE 2 /* lane per node, pair costs in registers, all C(8,k) subsets per pair */
#define KGPU_VARIANT_MEMO_BY_K 3     /* global best[k] computed once, pods look it up (what AUTO does; dense K1m for min_mem pods) */
#define KGPU_VARIANT_SPARSE 5        /* PER-PAIR work (north_star): lane per node, nodes ordered by free-GPU count, every pod
                                      * enumerates the k-subsets of the node's free positions; bench.py's headline      */
#define KGPU_VARIANT_TILE_MEMO 4     /* lane per node, per-k minima hoisted out of the pod loop (NOT the headline) */

#define KGPU_KEY_COST(key) ((uint32_t)((key) >> 40))
#define KGPU_KEY_NODE(key) ((uint32_t)(((key) >> 8) & 0xFFFFFFFFu))
#define KGPU_KEY_MASK(key) ((uint32_t)((key)&0xFFu))

typedef struct kgpu_ctx kgpu_t;

/* "major.minor.patch" of the library. */
const char *kgpu_version(void);

/* Create a scorer on CUDA device(s) dev_ids[0..ndev).  ndev == 1: one handle per
 * GPU (one process per GPU, or several handles in one process).  ndev > 1: the
 * handle shards the node array over the devices and combines their results
 * (single scheduler process driving all local GPUs). */
int kgpu_create(const int *dev_ids, int ndev, kgpu_t **out);
int kgpu_destroy(kgpu_t *h);

/* Message of the last failing call on h (or on this thread if h == NULL). */
const char *kgpu_last_error(kgpu_t *h);

/* Link-level -> cost table, 16 entries, each 0..KGPU_MAX_WEIGHT.
 * Default {64,32,16,8,4,2,1,0,...}: level 1 (cross-CPU) costs most, NVLink 0. */
int kgpu_set_weights(kgpu_t *h, const int32_t w[KGPU_NUM_LEVELS]);
int kgpu_get_weights(kgpu_t *h, int32_t w[KGPU_NUM_LEVELS]);

int kgpu_set_variant(kgpu_t *h, int variant);

/* Replace the node array (host pointers).  node_id_base is added to the local
 * index to form the node_id field of the keys (global id of this shard's node 0). */
int kgpu_upload_nodes(kgpu_t *h, const int32_t *topo, const int32_t *free_mask, int64_t n,
                      int64_t node_id_base);
/* Per-GPU memory (MiB) of every node, n = kgpu_num_nodes entries of 8.  Until this is called every
 * GPU has unlimited memory, i.e. the pods' min_mem_mib never excludes anything.  A later
 * kgpu_upload_nodes resets it to unlimited. */
int kgpu_upload_gpu_memory(kgpu_t *h, const int32_t *mem_mib, int64_t n);
int kgpu_update_gpu_memory(kgpu_t *h, int64_t idx, const int32_t mem_mib[8]);
/* Overwrite one node (AddNode on an existing name / usage update). */
int kgpu_update_node(kgpu_t *h, int64_t idx, const int32_t topo[64], int32_t free_mask);
int kgpu_set_free_mask(kgpu_t *h, int64_t idx, int32_t free_mask);
/* The same for n nodes in one call (a scheduling cycle's TakePodResources / ReturnPodResources,
 * gpu_scheduler.go:57-63): one host-to-device copy and one kernel that stores the masks and refreshes the
 * scorer's cached records of exactly those nodes.  A node listed twice gets its LAST mask. */
int kgpu_set_free_masks(kgpu_t *h, const int64_t *idx, const int32_t *free_mask, int64_t n);
/* RemoveNode: the slot stays, its GPUs become unschedulable (free_mask = 0). */
int kgpu_remove_node(kgpu_t *h, int64_t idx);
int64_t kgpu_num_nodes(kgpu_t *h);

/* Score P pods against every node: host buffers in, host buffers out
 * (H2D copy of pods + kernel(s) + D2H copy of keys, synchronous). */
int kgpu_score_batch(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys);

/* Same with device buffers on the handle's device (ndev == 1 handles only),
 * enqueued on `stream` (a cudaStream_t; NULL = the CUDA default stream, as in every CUDA
 * API), no sync.  The node array must not be changed until the work has completed.
 * d_pods must be 16-byte aligned. */
int kgpu_score_batch_device(kgpu_t *h, const int32_t *d_pods, int64_t P, uint64_t *d_keys,
                            void *stream);

/* Same, with promises about the batch the device-buffer path cannot check for itself:
 * KGPU_BATCH_NO_MIN_MEM = no pod of this batch has min_mem_mib > 0 (skips the flag kernel and the
 * K1m launch whose blocks would only read the flag and exit). */
#define KGPU_BATCH_NO_MIN_MEM 1
int kgpu_score_batch_device_ex(kgpu_t *h, const int32_t *d_pods, int64_t P, uint64_t *d_keys, void *stream,
                               int batch_flags);

/* Per-pair query (one PodFitsDevice(node, pod) call, or a list of them): for each i,
 * out_node_keys[i] = (cost << 8) | gpu_mask of the cheapest k[i]-subset of the free GPUs
 * of node node_idx[i] (local index as uploaded), or UINT32_MAX if it does not fit.
 * min_mem_mib may be NULL (no memory requirement) or hold one requirement per pair.
 * Host buffers, synchronous. */
int kgpu_score_pairs(kgpu_t *h, const int64_t *node_idx, const int32_t *k, const int32_t *min_mem_mib, int64_t n,
                     uint32_t *out_node_keys);

/* The (node, k) fit table: for every node and k = 0..8 the (cost << 8) | gpu_mask of its cheapest k-subset of
 * free GPUs (UINT32_MAX: does not fit), computed by one launch and kept as a host copy inside the handle.
 * kgpu_fit_lookup reads that copy -- no launch, no copy: this is what serves PodFitsDevice, which the core calls
 * once per (node, pod) pair (gpu_scheduler.go:34-44).  The table is built on first use and kept current by
 * kgpu_update_node / kgpu_set_free_mask(s) (they refresh the rows of the nodes they touch); kgpu_upload_nodes,
 * kgpu_set_weights and kgpu_place_batch invalidate it (rebuilt on the next lookup).  kgpu_build_fit_table
 * forces the build (e.g. at the start of a scheduling cycle).  kgpu_score_pairs uses the same table for pairs
 * without a memory requirement. */
int kgpu_build_fit_table(kgpu_t *h);
int kgpu_fit_lookup(kgpu_t *h, int64_t node_idx, int32_t k, uint32_t *out_node_key);

/* Stateful sequential placement (what TakePodResources would make of a scheduling cycle;
 * a no-op in the reference, gpu_scheduler.go:57-63).  Pods are placed IN ORDER; each one gets
 * the best (cost, node, mask) under the free masks left by the pods before it and then takes
 * those GPUs: the handle's device-side free masks are updated.  min_mem_mib is honoured like
 * in kgpu_score_batch; one batch may carry at most 7 distinct positive min_mem_mib values
 * (KGPU_ERR_INVALID otherwise).  Host buffers, synchronous, single-device handles only. */
int kgpu_place_batch(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys);
/* Same with flags.  KGPU_PLACE_DRY_RUN: the pods are placed in order on a scratch copy of the free masks, so
 * the keys are conflict-free PROPOSALS for the whole batch (no two pods share a GPU) while the handle's state
 * is untouched; commit the accepted ones with kgpu_set_free_masks (TakePodResources). */
#define KGPU_PLACE_DRY_RUN 1
int kgpu_place_batch_ex(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys, int flags);
/* Same with gangs: pods that only work together (the workers of one distributed training job) are placed all or
 * nothing.  gang[P] holds one id per pod: 0 = the pod is on its own; a GANG is a maximal run of consecutive pods with
 * the same nonzero id, so list each gang's members next to each other (an id that appears in two separate runs is
 * KGPU_ERR_INVALID, checked before anything runs).  Pods are placed in order as by kgpu_place_batch_ex; when a member
 * does not fit (or asks for k outside 0..8), the members of its gang placed before it give their GPUs back, the
 * members after it are not tried, and every member of the gang gets KGPU_NO_FIT: the free masks are exactly as they
 * were before the gang's first member, and the pods after the gang see that state.  The result equals
 * kgpu_place_batch_ex on the batch with every failed gang deleted.  Members may differ in k and min_mem_mib.
 * gang == NULL is kgpu_place_batch_ex.  Flags, min_mem_mib limits and single-device handles as there. */
int kgpu_place_batch_gang(kgpu_t *h, const int32_t *pods, const int32_t *gang, int64_t P, uint64_t *out_keys, int flags);
/* Gangs inside one network domain.  For a multi-node job the inter-node network carries the all-reduce, so where the
 * members sit relative to each other matters as much as the GPUs inside each node.
 *
 * Each node has a DOMAIN: -1 (none) or an id 0 <= d < n (n = kgpu_num_nodes).  A domain is the set of nodes under one
 * leaf switch, one InfiniBand scalable unit or one NVLink Switch domain; the caller decides.  kgpu_upload_domains sets
 * the whole table (n entries; a value outside -1..n-1 is KGPU_ERR_INVALID and leaves the table unchanged).  Until the
 * first upload every node's domain is -1; kgpu_upload_nodes resets the table to all -1, and kgpu_update_node,
 * kgpu_set_free_mask(s) and kgpu_remove_node leave it alone.  Scoring ignores domains, so an upload invalidates nothing.
 *
 * Each pod has a gang_domain value: 0 (no constraint), KGPU_GANG_DOMAIN_REQUIRED or KGPU_GANG_DOMAIN_PREFERRED.  Pods
 * are taken in order on the working masks F exactly as by kgpu_place_batch_gang, and pods and gangs with gang_domain 0
 * are placed exactly as there.  A CONSTRAINED gang has members m1..mj, consecutive pods with the same nonzero gang id,
 * all carrying the same nonzero gang_domain.  It is placed like this:
 *   1. Trial per domain.  For every domain d with at least one node, a trial on a copy F_d of F: for i = 1..j, if
 *      k(m_i) is outside 0..8 the trial fails; otherwise key_i = the minimum of (cost << 40 | node_id << 8 | S) over
 *      the nodes n with domain[n] = d, under F_d, with m_i's min_mem_mib applied as in scoring; if key_i is KGPU_NO_FIT
 *      the trial fails, otherwise F_d[n] &= ~S.  A trial that places every member has C_d = the sum of the members'
 *      costs.  A k = 0 member costs 0, takes nothing and gets the domain's lowest node.
 *   2. Choice.  If some trial succeeded, the gang takes the domain d* with the smallest (C_d, d): F = F_d*, and the
 *      members get that trial's keys.
 *   3. No domain fits, REQUIRED: every member gets KGPU_NO_FIT, and F is unchanged.
 *   4. No domain fits, PREFERRED: the gang is placed exactly as kgpu_place_batch_gang would place it on F: over all
 *      nodes, all or nothing.
 * So gang_domain == NULL (or all 0) is kgpu_place_batch_gang; with every node in domain 0, REQUIRED and PREFERRED both
 * are kgpu_place_batch_gang; the members of a placed REQUIRED gang sit in one domain, never on a node of domain -1; and a
 * PREFERRED gang gets the REQUIRED result when some domain fits, the plain gang result otherwise.
 * KGPU_ERR_INVALID, checked before anything runs: a gang_domain value outside {0, 1, 2}, a nonzero value on a pod with
 * gang id 0, members of one gang that disagree, a constrained gang of more than 37 000 members (the trials sum their
 * costs in 32 bits), and the checks of kgpu_place_batch_gang.  Flags (KGPU_PLACE_DRY_RUN) as there.  Both calls need
 * a single-device handle (KGPU_ERR_STATE otherwise).  Host buffers, synchronous. */
#define KGPU_GANG_DOMAIN_REQUIRED 1
#define KGPU_GANG_DOMAIN_PREFERRED 2
int kgpu_upload_domains(kgpu_t *h, const int32_t *domain, int64_t n);
int kgpu_place_batch_gang_domain(kgpu_t *h, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain,
                                 int64_t P, uint64_t *out_keys, int flags);
/* Nested network domains.  Fabrics have several levels: an NVLink or leaf-switch rack inside an InfiniBand spine or
 * scalable unit inside a pod.  A distributed job wants the smallest of them that holds it.
 *
 * kgpu_upload_domain_levels sets a table of `levels` (1..KGPU_MAX_DOMAIN_LEVELS) levels, domain[l * n + i] = node i's
 * domain at level l: -1 (none) or an id 0..n-1, ids separate at each level.  Level 0 is the finest (a rack), level
 * levels - 1 the coarsest.  The levels must nest: for a node i with domain[l][i] >= 0 and l + 1 < levels,
 * domain[l + 1][i] >= 0, and all nodes of one level-l domain have the same level-(l + 1) domain.  A node may have no
 * level-l domain and still have a level-(l + 1) one.  A value out of range, a nesting violation (the message names the
 * level, the node and the two ids) or `levels` outside 1..4 is KGPU_ERR_INVALID and leaves the table unchanged.
 * kgpu_upload_domains(h, d, n) is the one-level table.  Lifetime as for kgpu_upload_domains: before the first upload
 * and after kgpu_upload_nodes the table has one level with every node at -1; mask and node updates leave it alone.
 * kgpu_place_batch_gang_domain and kgpu_preempt_plan_gang_domain read level 0 and nothing else, so on a one-level table
 * they are what they always were.
 *
 * kgpu_place_batch_gang_levels: kgpu_place_batch_gang_domain with gang_level[P], the highest level each constrained
 * gang may span, 0..levels-1 (NULL = all 0).  The policy is TIGHTEST NETWORK DOMAIN FIRST, THEN GPU LINK COST.  A
 * constrained gang with bound r is placed on the working masks F like this:
 *   1. For l = 0, 1, ..., r: step 1 of kgpu_place_batch_gang_domain (one trial per non-empty domain) over the level-l
 *      domains, on F.  The first level with a successful trial wins: the gang takes that level's domain with the
 *      smallest (C_d, d), F = F_d and the members get that trial's keys.  A k = 0 member gets the domain's lowest node.
 *   2. No domain of any level <= r fits: REQUIRED gives every member KGPU_NO_FIT and leaves F unchanged; PREFERRED
 *      places the gang as kgpu_place_batch_gang would, over all nodes, all or nothing.
 * Pods and gangs with gang_domain 0 are placed exactly as by kgpu_place_batch_gang.  Consequences:
 *   Q1 gang_level NULL or all 0 is kgpu_place_batch_gang_domain, on level 0, with the same kernel launches;
 *   Q2 kgpu_place_batch_gang_domain after a multi-level upload equals the same call after uploading level 0 alone;
 *   Q3 with every node in level-1 domain 0, REQUIRED with r = 1 equals PREFERRED with r = 0;
 *   Q4 the members of a placed REQUIRED gang share one domain at some level l* <= r, never -1, and for every l < l*
 *      the gang alone with bound l gets KGPU_NO_FIT on the same state;
 *   Q5 PREFERRED gives the REQUIRED result when that places the gang, the plain gang result otherwise;
 *   Q6 a failed REQUIRED gang leaves F as it was.
 * KGPU_ERR_INVALID, checked before anything runs: every check of kgpu_place_batch_gang_domain, a gang_level outside
 * 0..levels-1 on a constrained pod, a nonzero gang_level on a pod with gang_domain 0, and members of one gang that
 * disagree on gang_level.  Flags (KGPU_PLACE_DRY_RUN) as there.  Both calls need a single-device handle
 * (KGPU_ERR_STATE otherwise).  Host buffers, synchronous.
 * Cost: a constrained gang runs one trial launch per level it climbs (a launch above the winning level exits at once).
 * A trial walks each domain with one warp.  On levels of small domains (at most 256 nodes) it reads 32 nodes per step;
 * on levels with a larger domain it reads the minima of 32-node chunks, 32 chunks per step, built once per level by one
 * extra launch, and rescans node by node only the chunks the trial itself has changed. */
#define KGPU_MAX_DOMAIN_LEVELS 4
int kgpu_upload_domain_levels(kgpu_t *h, const int32_t *domain, int levels, int64_t n);
int kgpu_place_batch_gang_levels(kgpu_t *h, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain,
                                 const int32_t *gang_level, int64_t P, uint64_t *out_keys, int flags);
/* Preemption (kube-scheduler's PostFilter for GPU pods): for a pod that fits nowhere, the node, GPUs and
 * lowest-priority running pods to evict.  No reference counterpart (DeviceScheduler has no preemption hook,
 * gpu_scheduler.go:21-71).  Single-device handles only (KGPU_ERR_STATE otherwise).
 *
 * The HOLDER TABLE holds one row of 8 int32 per node (laid out like gpu_mem): for GPU slot i, -1 (the GPU cannot be
 * evicted) or level << 3 | owner, with level 0..15 the priority level of the running pod that holds the GPU and owner
 * 0..7 that pod's number on this node.  All GPUs with the same owner on a node belong to one pod, are evicted
 * together and must carry the same level.  The entry of a free GPU (bit set in free_mask) is ignored.
 *   kgpu_upload_holders   sets the whole table (n = kgpu_num_nodes rows).
 *   kgpu_set_holders      replaces n rows (node indices idx[n], rows holders[n][8]) in one copy; a node listed
 *                         twice gets its LAST row.
 * An entry that is neither -1 nor 0..127, or an owner with two levels in one row, is KGPU_ERR_INVALID and leaves the
 * table unchanged.  The table's device memory (32 B per node) is allocated by the first upload.  kgpu_upload_nodes
 * resets the table to all -1; kgpu_update_node and kgpu_set_free_mask(s) leave it alone, so the caller keeps it in
 * step with the masks.
 *
 * kgpu_preempt_batch: pods[P][4] as for kgpu_score_batch, lvl[P] each pod's level 0..15 (KGPU_ERR_INVALID
 * otherwise).  For pod p, GPU i of node n is AVAILABLE if it is free, or if its entry is not -1 and its holder's
 * level is < lvl[p]; either way it must pass min_mem_mib as in scoring.  A candidate is (n, S) with S a k-subset of
 * available GPUs; its victims V(S) are the owners of the GPUs of S that are not free.  Candidates are ordered by
 * (max level in V, |V|, cost(S), node id, S), smallest first, an empty V before every non-empty one.
 *   out_keys[p]     the winner's key in the standard format, or KGPU_NO_FIT (no candidate, or k outside 0..8);
 *   out_victims[p]  bit o = owner o of the winner's node is evicted; 0 when nothing is.
 * So a pod that fits without eviction gets exactly its kgpu_score_batch key and victims 0, a level-0 pod never evicts,
 * and without a holder table the call equals kgpu_score_batch.  Snapshot semantics: nothing is evicted or taken, and
 * two pods of one batch may name the same victims.  Host buffers, synchronous. */
int kgpu_upload_holders(kgpu_t *h, const int32_t *holders, int64_t n);
int kgpu_set_holders(kgpu_t *h, const int64_t *idx, const int32_t *holders, int64_t n);
int kgpu_preempt_batch(kgpu_t *h, const int32_t *pods, const int32_t *lvl, int64_t P, uint64_t *out_keys,
                       uint32_t *out_victims);
/* kgpu_preempt_plan: the conflict-free counterpart of kgpu_preempt_batch, as kgpu_place_batch_ex(KGPU_PLACE_DRY_RUN)
 * is of kgpu_score_batch.  Arguments, output format and validation as for kgpu_preempt_batch.  A working state (F, H)
 * starts as the handle's free masks and holder table (all -1 if none was uploaded), and the pods are taken IN ORDER:
 * pod p gets what kgpu_preempt_batch would give it alone on (F, H); if it fits on node n with GPUs S and victims V,
 * then with R = the non-free GPUs of n whose owner is in V,  F[n] = (F[n] | R) & ~S  (the victims' GPUs that p does
 * not take are free for later pods) and H[n][g] = -1 for every g in S | R.  Consequences:
 *   - a pod of the batch is never a victim: GPUs the batch takes are marked -1, so a later pod of a higher level
 *     cannot evict an earlier one (as in kube-scheduler, where nominated pods are not preemption victims) -- pass the
 *     pods in priority order;
 *   - victim bits name owners of the holder table as it was at the call (nothing is renumbered or added);
 *   - the victim sets of different pods are disjoint, and so are the GPU sets of pods on one node;
 *   - P = 1 equals kgpu_preempt_batch; without a holder table, or with every lvl 0, the keys equal
 *     kgpu_place_batch_ex(KGPU_PLACE_DRY_RUN) and every victim mask is 0.
 * DRY RUN ONLY: the handle's free masks, holder table and caches are untouched.  Victims terminate asynchronously,
 * so a plan is committed by the caller, with kgpu_set_free_masks and kgpu_set_holders, once they are gone.
 * Limits (KGPU_ERR_INVALID, checked before anything runs; pods with k outside 0..8 do not count): at most 7 distinct
 * positive min_mem_mib values, and at most 32 distinct (level, min_mem_mib) pairs among the pods with level > 0.
 * Single-device handles only (KGPU_ERR_STATE otherwise).  Host buffers, synchronous. */
int kgpu_preempt_plan(kgpu_t *h, const int32_t *pods, const int32_t *lvl, int64_t P, uint64_t *out_keys,
                      uint32_t *out_victims);
/* kgpu_preempt_plan with gangs: the members of a gang (a multi-pod training job) evict their victims and take their
 * GPUs all together, or not at all.  gang[P] as for kgpu_place_batch_gang: 0 = the pod is on its own, a GANG is a
 * maximal run of consecutive pods with the same nonzero id, and an id that appears in two separate runs is
 * KGPU_ERR_INVALID (checked before anything runs).  Pods are taken in order on (F, H) exactly as by kgpu_preempt_plan.
 * When a member gets no candidate, or asks for k outside 0..8:
 *   - the members of its gang taken before it are undone, last first: each member's node gets back the free mask and
 *     holder row it had just before that member's update, so the victims they named are running pods again and later
 *     pods of the batch may name them;
 *   - the members after it are not tried;
 *   - every member of the gang gets KGPU_NO_FIT and victims 0.
 * The result equals kgpu_preempt_plan on the batch with every failed gang deleted.  Members may differ in k, level and
 * min_mem_mib; a k = 0 member fits and takes nothing.  gang == NULL is kgpu_preempt_plan.  Dry run only, limits,
 * single-device handles, host buffers and synchronous, as for kgpu_preempt_plan. */
int kgpu_preempt_plan_gang(kgpu_t *h, const int32_t *pods, const int32_t *lvl, const int32_t *gang, int64_t P,
                           uint64_t *out_keys, uint32_t *out_victims);
/* kgpu_preempt_plan_gang inside one network domain: a constrained gang evicts and takes its GPUs within one domain of
 * kgpu_upload_domains, so a plan never kills running pods for a gang that placement would then refuse.  Arguments,
 * output format, limits and dry-run semantics as for kgpu_preempt_plan_gang; gang_domain[P] as for
 * kgpu_place_batch_gang_domain (0, KGPU_GANG_DOMAIN_REQUIRED or KGPU_GANG_DOMAIN_PREFERRED); the domain table and its
 * lifetime as there.  (F, H) starts as the handle's free masks and holder table, and the pods are taken in order.  Pods
 * and gangs with gang_domain 0 are taken exactly as by kgpu_preempt_plan_gang.  A CONSTRAINED gang m1..mj:
 *   1. Trial per domain.  Every domain d with at least one node gets a trial on a copy (F_d, H_d): for i = 1..j, if
 *      k(m_i) is outside 0..8 the trial fails; a k = 0 member costs 0, evicts nothing, takes nothing and gets the
 *      domain's lowest node; otherwise m_i gets what kgpu_preempt_batch would give it alone on (F_d, H_d) restricted to
 *      the nodes with domain[n] = d (the minimum candidate in the order (max victim level, |V|, cost, node id, S), with
 *      min_mem_mib applied as in scoring); with no candidate the trial fails, otherwise the update rule of
 *      kgpu_preempt_plan is applied to (F_d, H_d).  A trial that places every member has the score (L_d, V_d, C_d):
 *      L_d the largest victim level over the members that evict (0 if none does), V_d the total victim count (victim
 *      sets are disjoint), C_d the sum of the members' costs.  So a trial that evicts nothing ranks before one that
 *      evicts level-0 pods.
 *   2. Choice.  If some trial succeeded, the gang takes the domain with the smallest (L_d, V_d, C_d, d): (F, H) becomes
 *      that trial's (F_d, H_d), and the members get its keys and victims.
 *   3. No domain fits, REQUIRED: every member gets KGPU_NO_FIT and victims 0; (F, H) is unchanged.
 *   4. No domain fits, PREFERRED: the gang is taken exactly as kgpu_preempt_plan_gang would take it on (F, H): over all
 *      nodes, all or nothing.
 * Consequences: P1 gang_domain == NULL (or all 0) is kgpu_preempt_plan_gang, with the same kernel launches; P2 with
 * every node in domain 0, REQUIRED and PREFERRED both are kgpu_preempt_plan_gang; P3 without a holder table, or with
 * every lvl 0, the keys equal kgpu_place_batch_gang_domain(KGPU_PLACE_DRY_RUN) on the same domain table and every
 * victim mask is 0; P4 the members of a placed REQUIRED gang and all their victims sit on the nodes of one domain,
 * never on a node of domain -1; P5 PREFERRED gives the REQUIRED result when some domain fits, the plain gang result
 * otherwise; P6 a failed REQUIRED gang leaves (F, H) as it was, so the result equals the call on the batch with that
 * gang deleted.
 * KGPU_ERR_INVALID, checked before anything runs: the checks of kgpu_preempt_plan_gang and the gang_domain checks of
 * kgpu_place_batch_gang_domain (values, members that agree, at most 37 000 members per constrained gang).  Dry run
 * only; single-device handles (KGPU_ERR_STATE otherwise).  Host buffers, synchronous. */
int kgpu_preempt_plan_gang_domain(kgpu_t *h, const int32_t *pods, const int32_t *lvl, const int32_t *gang,
                                  const int32_t *gang_domain, int64_t P, uint64_t *out_keys, uint32_t *out_victims);
/* Copy the current free masks (n = kgpu_num_nodes entries) back to the host. */
int kgpu_get_free_masks(kgpu_t *h, int32_t *out_free_mask, int64_t n);

/* K2: d_out[p] = min over g < G of d_gathered[g*P + p] (after an all-gather of
 * every shard's keys), enqueued on `stream`. */
int kgpu_reduce_shards_device(kgpu_t *h, const uint64_t *d_gathered, int G, int64_t P,
                              uint64_t *d_out, void *stream);

/* Peer-memory key exchange for the one-process-per-GPU launch (replaces the all-gather + kgpu_reduce_shards_device pair;
 * no reference counterpart, SURVEY.md 8(e)).  Every rank:
 *   kgpu_exchange_init(h, world, rank, max_pods, handle)   allocate the rank's slot/flag memory, export it
 *   <all-gather the KGPU_IPC_HANDLE_BYTES-byte handles through the launcher, e.g. torch.distributed>
 *   kgpu_exchange_connect(h, handles)                      map every peer's memory (handles = [world][64])
 *   kgpu_score_batch_exchange(h, d_pods, P, &d_final, stream, flags)   per step, TWO launches: K1 on the local shard, then
 *       one kernel that stores the P bests into every rank's slot array over NVLink (plain coalesced stores), meets the
 *       other ranks at a flag barrier in peer memory and takes the per-pod minimum over the G slots.  *d_final (device
 *       memory owned by the handle, valid until the next-but-one call) then holds the global keys on every rank.
 *   kgpu_exchange_barrier(h, stream)                       the same kernel with P = 0: a device-side barrier of the ranks
 * All ranks must make the same sequence of exchange calls.  A rank that waits more than ~10 s for its peers raises an
 * error (reported as KGPU_ERR_COMM by a later call) instead of hanging the GPU.  Single-device handles only. */
#define KGPU_IPC_HANDLE_BYTES 64
int kgpu_exchange_init(kgpu_t *h, int world, int rank, int64_t max_pods, unsigned char *out_handle);
int kgpu_exchange_connect(kgpu_t *h, const unsigned char *handles);
int kgpu_score_batch_exchange(kgpu_t *h, const int32_t *d_pods, int64_t P, const uint64_t **d_final_keys,
                              void *stream, int batch_flags);
int kgpu_exchange_barrier(kgpu_t *h, void *stream);

/* Number of CUDA kernels this handle has launched so far (bench bookkeeping). */
int64_t kgpu_kernel_launches(kgpu_t *h);
/* Wall-clock duration (ms) of the most recent kgpu_upload_nodes: host-to-device copies, the device-side
 * value-domain check, the K1s order (counting sort by free-GPU count) and the compacted records. */
double kgpu_last_upload_ms(kgpu_t *h);
/* Device duration (ms, CUDA events on the launching stream) of the K1 launch(es)
 * of the most recent kgpu_score_batch call. */
double kgpu_last_kernel_ms(kgpu_t *h);

#ifdef __cplusplus
}
#endif
#endif /* KGPU_H_ */
