// device_scheduler.h -- C++ mirror of the reference's scheduler-side plugin surface.
//
// The reference host language is Go (no Go toolchain in this image), so the host layer
// above the C ABI (include/kgpu.h) is written in C++ with the same names, argument
// meaning and error behaviour as the Go code it stands in for:
//
//   kubedevice::types::*            <- github.com/Microsoft/KubeDevice-API/pkg/types as USED by
//                                      the reference (SURVEY.md 8(b) "Types crossing the boundary")
//   gpuplugintypes::SortedTreeNode  <- gpuplugintypes/types.go:9-13, typeutils.go:10-93
//   gpuschedulerplugin::*           <- gpuschedulerplugin/gpu.go, gpu_scheduler.go
//   CreateDeviceSchedulerPlugin()   <- gpuschedulerplugin/plugin/gpuscheduler.go:8
//
// The tree cache / request translation is kept because the external core scheduler
// consumes the rewritten DevRequests (UsingGroupScheduler() == true in the reference).
// What is NEW is the score: PodFitsDevice's third return value, hard-coded 0.0 in the
// reference (gpu_scheduler.go:34-44), comes from the GPU scorer (K1), and ScoreBatch()
// is the batched side-door that amortises the cgo/launch cost over a whole scheduling
// cycle (SURVEY.md 7 "Hard parts": cgo).
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

struct kgpu_ctx;

namespace kubedevice {
namespace types {

using ResourceName = std::string;
using ResourceList = std::map<ResourceName, int64_t>;          // ordered: SortedStringKeys for free
using ResourceLocation = std::map<ResourceName, ResourceName>;

extern const char *const DeviceGroupPrefix;                     // "resource/group"

struct ContainerInfo {
    ResourceList Requests, KubeRequests, DevRequests;
    ResourceLocation AllocateFrom;
};

struct PodInfo {
    std::string Name;
    ResourceList Requests;
    std::map<std::string, ContainerInfo> InitContainers, RunningContainers;
};

struct NodeInfo {
    std::string Name;   // present in KubeDevice-API's NodeInfo; the reference never reads it
    ResourceList Capacity, Allocatable, KubeCap, KubeAlloc;
};

void AddGroupResource(ResourceList &list, const std::string &key, int64_t val);   // gpu.go:50

}  // namespace types

namespace devicescheduler {
struct PredicateFailureReason {
    std::string reason;
};
}  // namespace devicescheduler
}  // namespace kubedevice

namespace gpuplugintypes {

extern const char *const ResourceGPU;   // "nvidia.com/gpu"  (gpuplugintypes/types.go:6)

struct SortedTreeNode {                 // gpuplugintypes/types.go:9-13
    int Val = 0;
    double Score = 0.0;
    std::vector<std::unique_ptr<SortedTreeNode>> Child;
};

SortedTreeNode *AddToSortedTreeNode(SortedTreeNode *node, int valToAdd);
SortedTreeNode *AddToSortedTreeNodeWithScore(SortedTreeNode *node, int valToAdd, double score);
void AddNodeToSortedTreeNode(SortedTreeNode *node, std::unique_ptr<SortedTreeNode> nodeToAdd);
bool CompareTreeNode(const SortedTreeNode *a, const SortedTreeNode *b);
std::string FormatTreeNode(const SortedTreeNode *node, int level = 0);   // PrintTreeNode's text

}  // namespace gpuplugintypes

namespace gpuschedulerplugin {

namespace types = kubedevice::types;
using gpuplugintypes::SortedTreeNode;

extern const char *const GPUTopologyGeneration;   // "gpu/gpu-generate-topology" (gpu_scheduler.go:14)
// Extension (no reference counterpart): pod-level request "every GPU I get must have at least this
// many MiB" -- checked against the per-GPU `<gpu>/memory` the node agent advertises.
extern const char *const GPUMinMemoryMiB;         // "gpu/gpu-min-memory-mib"
// Extension: pod-level request "I am one of a gang of pods that only work together" (e.g. the workers of one
// distributed training job).  Pods of one PlaceBatch / ProposeBatch call with the same nonzero value are placed all
// or nothing; 0 or absent = the pod is on its own.
extern const char *const GPUGangID;               // "gpu/gpu-gang-id"
// Extension: pod-level request "my gang wants one network domain" (SetNodeDomain): 1 = required (the gang is placed
// inside one domain or not at all), 2 = preferred (inside one domain if one fits, else as a plain gang), 0 or absent =
// no constraint.  Only on gang members, the same for every member of a gang; honoured by PlaceBatch and ProposeBatch
// (kgpu_place_batch_gang_domain).
extern const char *const GPUGangDomain;           // "gpu/gpu-gang-domain"
// Extension: pod-level request "my gang may span up to this level of nested domains" (SetNodeDomains: 0 = the finest
// level, e.g. a rack), default 0.  Only with GPUGangDomain, the same for every member of a gang; the gang takes the
// lowest level 0..this one with a domain that fits (kgpu_place_batch_gang_levels).  PlaceBatch and ProposeBatch honour
// it; PlanGangDomainPreemption refuses a nonzero value.
extern const char *const GPUGangDomainLevel;      // "gpu/gpu-gang-domain-level"
// Extension: pod-level request "my priority level", 0..15 (values outside are clamped), default 0.  PreemptBatch lets a
// pod evict running pods of a LOWER level; every placement records the level of its pod.
extern const char *const GPUPriorityLevel;        // "gpu/gpu-priority-level"

// ---- gpu.go, function for function ------------------------------------------------
types::ResourceList TranslateGPUResources(int64_t neededGPUs, const types::ResourceList &nodeResources,
                                          types::ResourceList containerRequests);
void SetGPUReqs(types::ContainerInfo &cont);
std::unique_ptr<SortedTreeNode> addToNode(std::unique_ptr<SortedTreeNode> node, const types::ResourceList &nodeResources,
                                          const std::string &partitionPrefix, const std::string &suffix, int partitionLevel);
double computeTreeScore(const SortedTreeNode *node);

// NodeCacheMap / NodeLocationMap (package globals in gpu.go:168-169) as an object.
class TreeCache {
public:
    struct Entry {
        std::unique_ptr<SortedTreeNode> tree;
        std::map<std::string, bool> ListOfNodes;
        double TreeScore = 0.0;
    };
    void AddResourcesToNodeTreeCache(const std::string &nodeName, const types::ResourceList &nodeResources);
    void RemoveNodeFromNodeTreeCache(const std::string &nodeName);
    // Deterministic where Go's map iteration is not: ties go to the shape that
    // compares smaller (same rule as the oracle).
    const SortedTreeNode *findBestTreeInCache(int num) const;
    const std::vector<std::unique_ptr<Entry>> &entries() const { return cache_; }
    const SortedTreeNode *location(const std::string &nodeName) const;

private:
    void removeNodeFromCache(const std::string &nodeName, const SortedTreeNode *loc);
    std::vector<std::unique_ptr<Entry>> cache_;
    std::map<std::string, const SortedTreeNode *> location_;
};

bool ConvertToBestGPURequests(const TreeCache &cache, types::PodInfo &podInfo);
// returns the error text ("" = nil) and `found`
std::string TranslatePodGPUResources(const TreeCache &cache, const types::NodeInfo &nodeInfo, types::PodInfo &podInfo,
                                     bool *found);

// ---- one GPU placement, as the kernels report it -------------------------------------
struct Placement {
    bool fits = false;
    uint32_t cost = 0;
    std::string nodeName;
    uint32_t gpuMask = 0;       // bit i = GPU slot i of that node
    uint64_t key = UINT64_MAX;  // raw (cost<<40 | node_id<<8 | mask)
    bool committed = false;     // the GPUs are already taken on the device (PlaceBatch) / by TakePodResources
    int level = 0;              // the pod's GPUPriorityLevel
};

// ---- gpu_scheduler.go: the DeviceScheduler boundary ------------------------------------
class NvidiaGPUScheduler {
public:
    // devices empty => host logic only (tree cache / translation); every scoring call
    // then fails loudly -- there is no CPU scorer in the product.
    // groupSchedulerMode = false (default): the plugin's own (node, GPU set) is authoritative -- PodAllocate fills
    //   AllocateFrom itself and UsingGroupScheduler() returns false, so the core does not run its group allocator
    //   over the rewritten DevRequests a second time (SURVEY.md 8(b): "return false iff it fills AllocateFrom").
    // groupSchedulerMode = true: the reference's contract (gpu_scheduler.go:69-71 returns true): PodAllocate only
    //   rewrites DevRequests (ConvertToBestGPURequests), AllocateFrom is left to the core's group allocator, and
    //   the GPU's score is advisory.
    explicit NvidiaGPUScheduler(const std::vector<int> &devices = {0}, bool groupSchedulerMode = false);
    ~NvidiaGPUScheduler();
    NvidiaGPUScheduler(const NvidiaGPUScheduler &) = delete;
    NvidiaGPUScheduler &operator=(const NvidiaGPUScheduler &) = delete;

    // The reference's eight methods (gpu_scheduler.go:21-71), same meaning.
    void AddNode(const std::string &nodeName, types::NodeInfo *nodeInfo);
    void RemoveNode(const std::string &nodeName);
    bool PodFitsDevice(types::NodeInfo *nodeInfo, types::PodInfo *podInfo, bool fillAllocateFrom,
                       std::vector<kubedevice::devicescheduler::PredicateFailureReason> *reasons, double *score);
    std::string PodAllocate(types::NodeInfo *nodeInfo, types::PodInfo *podInfo);              // "" = nil error
    std::string TakePodResources(types::NodeInfo *nodeInfo, types::PodInfo *podInfo);
    std::string ReturnPodResources(types::NodeInfo *nodeInfo, types::PodInfo *podInfo);
    std::string GetName() const { return "nvidiagpu"; }
    bool UsingGroupScheduler() const { return groupSchedulerMode_; }

    // Extensions (no reference counterpart).
    // Real NVML link matrix for a node (int32[8][8] row-major, levels 0..15) instead of the
    // one derived from its 2-level group names.
    std::string SetNodeTopology(const std::string &nodeName, const int32_t topo[64]);
    // The network domain of a node (the nodes under one leaf switch, one scalable unit or one NVLink Switch domain);
    // "" = none, the default.  Names map to dense ids in sorted order; the device table is re-uploaded before the next
    // PlaceBatch / ProposeBatch when a domain or the node array has changed.
    std::string SetNodeDomain(const std::string &nodeName, const std::string &domainName);
    // Nested network domains: names[l] is the node's domain at level l (0 = the finest, e.g. a rack inside a spine at
    // level 1), "" = none at that level.  Names map to dense ids per level in sorted order; the table has as many levels
    // as the longest list, and the levels must nest (kgpu_upload_domain_levels, checked at the next PlaceBatch).
    // SetNodeDomain(node, name) is SetNodeDomains(node, {name}).
    std::string SetNodeDomains(const std::string &nodeName, const std::vector<std::string> &names);
    // Node from the node agent's GPU inventory JSON (nvgputypes.GpusInfo): names exactly as the
    // agent would advertise them, then AddNode, then the REAL link matrix (not the one implied by
    // the two group levels).  Fills *nodeInfo like the agent's UpdateNodeInfo.  "" or error text.
    std::string AddNodeFromGpusInfo(const std::string &nodeName, const std::string &gpusInfoJSON, bool useNVML,
                                    types::NodeInfo *nodeInfo);
    // Score a whole scheduling cycle in one kernel launch: best node + GPU set per pod.  Gang ids and gang domains are
    // ignored: snapshot scores change no state, so there is nothing to keep all or nothing or together.
    std::string ScoreBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out);
    // Place a whole cycle IN ORDER on the device: each pod takes its GPUs before the next one is
    // scored (K3).  The placements are remembered like ScoreBatch's and the usage is recorded, so a
    // later PodAllocate / ReturnPodResources works on them.  Gangs (GPUGangID): every member is placed right after
    // the gang's first member in the batch (the others keep their order); if one member does not fit, the whole gang
    // gets fits = false, takes nothing, and the pods after it are placed as if it had not been in the batch.  A gang
    // whose members carry GPUGangDomain is placed inside the network domain where its members cost least in sum
    // (kgpu_place_batch_gang_domain has the definition); a member with a gang domain but no gang id, or members of one
    // gang that disagree, is an error.  `out` is in the caller's order.
    std::string PlaceBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out);
    // Conflict-free PROPOSALS for a whole cycle: like PlaceBatch (each pod sees the GPUs the pods before it would
    // take) but on a scratch copy of the device state -- nothing is taken until TakePodResources commits a pod.
    // This is the conflict resolution ScoreBatch lacks: its snapshot scores hand every pod of equal k the same GPUs.
    // Gangs as in PlaceBatch.
    std::string ProposeBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out);
    // Preemption (kube-scheduler's PostFilter): for each pod, the best placement when running pods of a lower
    // GPUPriorityLevel may be evicted -- fewest and lowest-level victims first (lowest highest victim level, then fewest
    // victims, then cost, node, GPUs), see kgpu_preempt_batch.  A pod that fits without eviction gets its ScoreBatch
    // placement and no victims.  (*victims)[p] names the running pods to evict, in name order.  The running pods are the
    // committed placements (PlaceBatch, TakePodResources) until ReturnPodResources; GPUs in use that no committed
    // placement accounts for are never evicted.  Snapshot semantics: nothing is evicted, taken or remembered, two pods
    // may name the same victims, and gang ids and gang domains are ignored.
    std::string PreemptBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                             std::vector<std::vector<std::string>> *victims);
    // The conflict-free counterpart of PreemptBatch, as ProposeBatch is of ScoreBatch (kgpu_preempt_plan): pods are
    // taken in the caller's order, each on the state the pods before it leave -- their GPUs taken, their victims' GPUs
    // free, neither evictable again -- so no two pods name the same victim or GPU.  Pass pods in priority order.  Like
    // PreemptBatch, nothing is evicted, taken or remembered and gang ids and gang domains are ignored: commit a plan with
    // TakePodResources / ReturnPodResources once the victims are gone.
    std::string PlanPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                               std::vector<std::vector<std::string>> *victims);
    // PlanPreemption with gangs (GPUGangID, kgpu_preempt_plan_gang): members are moved up to their gang's first member
    // as in PlaceBatch, and a gang evicts and takes all together or not at all.  If one member cannot be placed, the
    // whole gang gets fits = false and no victims, and the pods after it see the victims its other members would have
    // named as running pods again.  Gang domains are ignored.  `out` and `victims` are in the caller's order.
    std::string PlanGangPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                   std::vector<std::vector<std::string>> *victims);
    // PlanGangPreemption inside one network domain (kgpu_preempt_plan_gang_domain): a gang whose members carry
    // GPUGangDomain evicts and takes its GPUs inside the domain (SetNodeDomain) whose plan is best in (highest victim
    // level, victim count, summed cost, domain id); with none, a required gang gets fits = false and no victims, a
    // preferred one is planned as by PlanGangPreemption.  The domain table is pushed as for PlaceBatch, members move
    // up to their gang's first member, and bad gang domains are errors as there.  Nothing is taken or remembered.
    std::string PlanGangDomainPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                         std::vector<std::vector<std::string>> *victims);
    std::string LastError() const { return lastError_; }
    const TreeCache &cache() const { return cache_; }
    bool hasDevice() const { return handle_ != nullptr; }

    struct NodeRecord {                       // what AddNode learned about a node
        std::string name;
        int64_t index = -1;                   // slot in the device-side node array
        int nGpus = 0;
        std::vector<std::string> gpuNames;    // slot -> "gpugrp1/a/gpugrp0/b/gpu/<id>"
        int32_t topo[64] = {0};
        int32_t memMiB[8] = {0};              // per slot, from the advertised <gpu>/memory (0 = unknown)
        bool hasMem = false;
        uint32_t presentMask = 0, usedMask = 0;
        bool explicitTopo = false;
        bool removed = false;
        std::vector<std::string> owners;      // holder-table owner o -> pod name, as last pushed to the device
        std::vector<std::string> domains;     // SetNodeDomains: per level, "" = none
    };
    const NodeRecord *node(const std::string &nodeName) const;
    static int64_t PodGPUCount(const types::PodInfo &podInfo);     // k of gpu.go:295-303

private:
    std::string syncNode(const NodeRecord &rec);
    std::string flushNodes();
    std::string scoreOne(const NodeRecord &rec, int k, int32_t minMemMiB, uint32_t *nodeKey);
    enum class BatchMode { Snapshot, Sequential, DryRun, Preempt, PreemptPlan, PreemptGangPlan, PreemptGangDomainPlan };
    std::string runBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out, BatchMode mode,
                         std::vector<std::vector<std::string>> *victims = nullptr);
    const NodeRecord *recordOf(const types::NodeInfo *nodeInfo) const;
    std::string pushMask(NodeRecord &rec);
    std::string pushHolders();
    std::string pushDomains();
    TreeCache cache_;
    std::map<std::string, NodeRecord> nodes_;
    std::vector<std::string> indexToName_;
    std::map<std::string, Placement> lastPlacement_;   // pod name -> ScoreBatch result
    std::map<const types::NodeInfo *, std::string> infoToName_;   // AddNode's NodeInfo* -> node name
    kgpu_ctx *handle_ = nullptr;
    bool dirty_ = false;                                // node COUNT changed: the device array must be re-uploaded
    std::vector<std::string> changed_;                  // existing nodes whose matrix / presence changed (kgpu_update_node)
    std::set<std::string> holdersChanged_;              // nodes whose running pods changed since the last holder push
    bool holdersReset_ = true;                          // the device table was reset (re-upload): push every row
    bool domainsDirty_ = false;                         // a node's domain changed, or a re-upload reset the device table
    bool groupSchedulerMode_ = false;
    std::string lastError_;
};

// gpuschedulerplugin/plugin/gpuscheduler.go:8 -- the factory symbol the core looks up.
std::unique_ptr<NvidiaGPUScheduler> CreateDeviceSchedulerPlugin(std::string *err);

}  // namespace gpuschedulerplugin
