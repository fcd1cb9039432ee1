// device_scheduler.cc -- see device_scheduler.h.  Citations are to /root/reference.
#include "device_scheduler.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <regex>

#include "../../../include/kgpu.h"
#include "gpus_info.h"

namespace kubedevice {
namespace types {
const char *const DeviceGroupPrefix = "resource/group";
void AddGroupResource(ResourceList &list, const std::string &key, int64_t val) {
    list[std::string(DeviceGroupPrefix) + "/" + key] = val;
}
}  // namespace types
}  // namespace kubedevice

// =====================================================================================
namespace gpuplugintypes {

const char *const ResourceGPU = "nvidia.com/gpu";

namespace {
// typeutils.go:10-23: first child that is smaller (Val, then Score); equal keys keep
// insertion order because the comparison is strict.
size_t insertionPoint(const SortedTreeNode *node, int val, double score) {
    size_t at = node->Child.size();
    for (size_t i = 0; i < node->Child.size(); i++) {
        const SortedTreeNode *c = node->Child[i].get();
        if (c->Val < val || (c->Val == val && c->Score < score)) {
            at = i;
            break;
        }
    }
    return at;
}
}  // namespace

SortedTreeNode *AddToSortedTreeNodeWithScore(SortedTreeNode *node, int valToAdd, double score) {
    auto fresh = std::make_unique<SortedTreeNode>();
    fresh->Val = valToAdd;
    fresh->Score = score;
    SortedTreeNode *raw = fresh.get();
    node->Child.insert(node->Child.begin() + (std::ptrdiff_t)insertionPoint(node, valToAdd, score), std::move(fresh));
    return raw;
}

SortedTreeNode *AddToSortedTreeNode(SortedTreeNode *node, int valToAdd) {
    return AddToSortedTreeNodeWithScore(node, valToAdd, 0.0);
}

void AddNodeToSortedTreeNode(SortedTreeNode *node, std::unique_ptr<SortedTreeNode> nodeToAdd) {
    const size_t at = insertionPoint(node, nodeToAdd->Val, nodeToAdd->Score);
    node->Child.insert(node->Child.begin() + (std::ptrdiff_t)at, std::move(nodeToAdd));
}

bool CompareTreeNode(const SortedTreeNode *a, const SortedTreeNode *b) {   // typeutils.go:75-93
    if (!a && !b) return true;
    if (!a || !b) return false;
    if (a->Val != b->Val || a->Child.size() != b->Child.size()) return false;
    for (size_t i = 0; i < a->Child.size(); i++)
        if (!CompareTreeNode(a->Child[i].get(), b->Child[i].get())) return false;
    return true;
}

std::string FormatTreeNode(const SortedTreeNode *node, int level) {        // typeutils.go:42-63
    std::string out(3 * (size_t)level, ' ');
    out += std::to_string(node->Val) + "\n";
    for (const auto &c : node->Child) out += FormatTreeNode(c.get(), level + 1);
    return out;
}

}  // namespace gpuplugintypes

// =====================================================================================
namespace gpuschedulerplugin {

using gpuplugintypes::ResourceGPU;

const char *const GPUTopologyGeneration = "gpu/gpu-generate-topology";
const char *const GPUMinMemoryMiB = "gpu/gpu-min-memory-mib";
const char *const GPUGangID = "gpu/gpu-gang-id";
const char *const GPUGangDomain = "gpu/gpu-gang-domain";
const char *const GPUGangDomainLevel = "gpu/gpu-gang-domain-level";
const char *const GPUPriorityLevel = "gpu/gpu-priority-level";

namespace {

int64_t getOr0(const types::ResourceList &l, const std::string &k) {
    auto it = l.find(k);
    return it == l.end() ? 0 : it->second;
}

// strconv.Atoi: optional sign, decimal digits only.
bool goAtoi(const std::string &s, int *out) {
    if (s.empty()) return false;
    size_t i = (s[0] == '+' || s[0] == '-') ? 1 : 0;
    if (i == s.size()) return false;
    long long v = 0;
    for (size_t j = i; j < s.size(); j++) {
        if (s[j] < '0' || s[j] > '9') return false;
        v = v * 10 + (s[j] - '0');
        if (v > std::numeric_limits<int>::max()) return false;
    }
    *out = (int)(s[0] == '-' ? -v : v);
    return true;
}

std::string escapeRegex(const std::string &s) {
    static const std::string meta = R"(\^$.|?*+()[]{})";
    std::string out;
    for (char c : s) {
        if (meta.find(c) != std::string::npos) out += '\\';
        out += c;
    }
    return out;
}

// UNPINNED: KubeDevice-API resource.TranslateResource is absent from the reference tree and
// no reference test reaches it; behaviour restated from gpu_scheduler.go:13,22-24 (see DESIGN.md
// "Unpinned pieces"): one fresh group index per distinct id, requests visited in sorted order.
bool TranslateResource(const types::ResourceList &nodeResources, types::ResourceList &containerRequests,
                       const std::string &thisStage, const std::string &nextStage) {
    const std::string ts = escapeRegex(thisStage), ns = escapeRegex(nextStage);
    const std::regex rxNode(".*/" + ts + "/(.*?)/" + ns + "/.*");
    bool needed = false;
    for (const auto &kv : nodeResources)
        if (std::regex_search(kv.first, rxNode)) { needed = true; break; }
    if (!needed) return false;
    const std::regex rxHas("(.*)/" + ts + "/(.*?)/" + ns + "/(.*?)/(.*)");
    const std::regex rxNeed("(.*)/" + ns + "/(.*?)/(.*)");
    int maxIdx = -1;
    std::smatch m;
    for (const auto &kv : containerRequests)
        if (std::regex_search(kv.first, m, rxHas)) {
            int v;
            if (goAtoi(m[2].str(), &v)) maxIdx = std::max(maxIdx, v);
        }
    std::map<std::string, int> groupOf;
    types::ResourceList out;
    bool modified = false;
    for (const auto &kv : containerRequests) {           // std::map iterates in sorted-key order
        if (std::regex_search(kv.first, rxHas)) { out[kv.first] = kv.second; continue; }
        if (!std::regex_search(kv.first, m, rxNeed, std::regex_constants::match_continuous)) { out[kv.first] = kv.second; continue; }
        const std::string ident = m[2].str();
        auto it = groupOf.find(ident);
        if (it == groupOf.end()) it = groupOf.emplace(ident, ++maxIdx).first;
        out[m[1].str() + "/" + thisStage + "/" + std::to_string(it->second) + "/" + nextStage + "/" + ident + "/" + m[3].str()] = kv.second;
        modified = true;
    }
    containerRequests.swap(out);
    return modified;
}

double goDiv(long long num, long long den) {             // float64(num)/float64(den), Go semantics
    if (den != 0) return (double)num / (double)den;
    if (num == 0) return std::numeric_limits<double>::quiet_NaN();
    return num > 0 ? std::numeric_limits<double>::infinity() : -std::numeric_limits<double>::infinity();
}

double computeTreeScoreAtLevel(const SortedTreeNode *node, int level, size_t numChild) {   // gpu.go:180-186
    double score = goDiv((long long)node->Val * level, (long long)numChild);
    for (const auto &c : node->Child) score += computeTreeScoreAtLevel(c.get(), level + 1, node->Child.size());
    return score;
}

// shape order used for the deterministic tie-break: (Val, children...) lexicographic
int compareShape(const SortedTreeNode *a, const SortedTreeNode *b) {
    if (a->Val != b->Val) return a->Val < b->Val ? -1 : 1;
    const size_t n = std::min(a->Child.size(), b->Child.size());
    for (size_t i = 0; i < n; i++) {
        const int c = compareShape(a->Child[i].get(), b->Child[i].get());
        if (c) return c;
    }
    if (a->Child.size() != b->Child.size()) return a->Child.size() < b->Child.size() ? -1 : 1;
    return 0;
}

// gpu.go:247-271
void assignGPUs(const SortedTreeNode *node, const std::string &prefix, const std::string &resourceGrp,
                const std::string &resource, const std::string &suffix, int level, int *numLeft,
                types::ResourceList *resList) {
    if (level == 0) {
        const int toTake = *numLeft <= node->Val ? *numLeft : node->Val;
        for (int i = 0; i < toTake; i++) (*resList)[prefix + "/" + resource + "/" + std::to_string(i) + "/" + suffix] = 1;
        *numLeft -= toTake;
        return;
    }
    for (size_t i = 0; i < node->Child.size(); i++) {
        std::string next = prefix + std::to_string(level - 1) + "/" + std::to_string(i);
        if (level - 1 != 0) next += "/" + resourceGrp;
        assignGPUs(node->Child[i].get(), next, resourceGrp, resource, suffix, level - 1, numLeft, resList);
    }
}

// gpu.go:273-291
void translateToTree(const SortedTreeNode *node, types::ContainerInfo *cont) {
    static const std::regex rxGpu(".*/gpu/.*");
    types::ResourceList kept;
    for (const auto &kv : cont->DevRequests)
        if (!std::regex_search(kv.first, rxGpu)) kept.insert(kv);
    cont->DevRequests.swap(kept);
    int numGPUs = (int)getOr0(cont->Requests, ResourceGPU);
    types::ResourceList res;
    assignGPUs(node, std::string(types::DeviceGroupPrefix) + "/gpugrp", "gpugrp", "gpu", "cards", 2, &numGPUs, &res);
    for (const auto &kv : res) cont->DevRequests[kv.first] = kv.second;
}

}  // namespace

// gpu.go:16-66
types::ResourceList TranslateGPUResources(int64_t neededGPUs, const types::ResourceList &nodeResources,
                                          types::ResourceList containerRequests) {
    static const std::regex rx(std::string(types::DeviceGroupPrefix) + ".*/gpu/(.*?)/cards");
    bool need = false;
    for (const auto &kv : nodeResources)
        if (std::regex_search(kv.first, rx)) { need = true; break; }
    if (!need) return containerRequests;
    int have = 0, maxIndex = -1;
    std::smatch m;
    for (const auto &kv : containerRequests)
        if (std::regex_search(kv.first, m, rx)) {
            have++;
            int idx;
            if (goAtoi(m[1].str(), &idx)) maxIndex = std::max(maxIndex, idx);
        }
    const int diff = (int)(neededGPUs - have);
    for (int i = 0; i < diff; i++)
        types::AddGroupResource(containerRequests, "gpu/" + std::to_string(maxIndex + i + 1) + "/cards", 1);
    TranslateResource(nodeResources, containerRequests, "gpugrp0", "gpu");
    TranslateResource(nodeResources, containerRequests, "gpugrp1", "gpugrp0");
    return containerRequests;
}

// gpu.go:80-92
void SetGPUReqs(types::ContainerInfo &cont) {
    auto a = cont.Requests.find(ResourceGPU);
    auto b = cont.KubeRequests.find(ResourceGPU);
    if (a != cont.Requests.end() && b != cont.KubeRequests.end()) a->second = std::max(a->second, b->second);
    else if (a != cont.Requests.end()) { /* keep */ }
    else if (b != cont.KubeRequests.end()) cont.Requests[ResourceGPU] = b->second;
    else cont.Requests[ResourceGPU] = 0;
}

// gpu.go:129-161
std::unique_ptr<SortedTreeNode> addToNode(std::unique_ptr<SortedTreeNode> node, const types::ResourceList &nodeResources,
                                          const std::string &partitionPrefix, const std::string &suffix, int partitionLevel) {
    const std::regex rx(".*/" + partitionPrefix + std::to_string(partitionLevel) + "/(.*?)/.*/" + suffix);
    std::map<std::string, types::ResourceList> childMap;
    int totalLen = 0;
    std::smatch m;
    for (const auto &kv : nodeResources)                     // sorted keys
        if (std::regex_search(kv.first, m, rx)) {
            childMap[m[1].str()][kv.first] = kv.second;
            totalLen++;
        }
    if (!node) {
        node = std::make_unique<SortedTreeNode>();
        node->Val = totalLen;
    }
    for (const auto &sub : childMap) {                       // sorted group ids
        auto child = std::make_unique<SortedTreeNode>();
        child->Val = (int)sub.second.size();
        if (partitionLevel > 0) {
            child = addToNode(std::move(child), sub.second, partitionPrefix, suffix, partitionLevel - 1);
            child->Score = computeTreeScore(child.get());   // gpu.go:155
        }
        gpuplugintypes::AddNodeToSortedTreeNode(node.get(), std::move(child));
    }
    return node;
}

double computeTreeScore(const SortedTreeNode *node) { return computeTreeScoreAtLevel(node, 0, node->Child.size()); }

// ---- TreeCache (gpu.go:163-245) -------------------------------------------------------
const SortedTreeNode *TreeCache::location(const std::string &nodeName) const {
    auto it = location_.find(nodeName);
    return it == location_.end() ? nullptr : it->second;
}

void TreeCache::removeNodeFromCache(const std::string &nodeName, const SortedTreeNode *loc) {
    if (!loc) return;
    for (size_t i = 0; i < cache_.size(); i++)
        if (cache_[i]->tree.get() == loc) {
            cache_[i]->ListOfNodes.erase(nodeName);
            if (cache_[i]->ListOfNodes.empty()) cache_.erase(cache_.begin() + (std::ptrdiff_t)i);
            return;
        }
}

void TreeCache::AddResourcesToNodeTreeCache(const std::string &nodeName, const types::ResourceList &nodeResources) {
    if (nodeResources.empty()) return;                                         // gpu.go:193-195
    std::unique_ptr<SortedTreeNode> node = addToNode(nullptr, nodeResources, "gpugrp", "cards", 1);
    const SortedTreeNode *loc = location(nodeName);
    if (gpuplugintypes::CompareTreeNode(node.get(), loc)) return;              // unchanged
    removeNodeFromCache(nodeName, loc);
    for (auto &e : cache_)
        if (gpuplugintypes::CompareTreeNode(node.get(), e->tree.get())) {
            e->ListOfNodes[nodeName] = true;
            location_[nodeName] = e->tree.get();
            return;
        }
    auto e = std::make_unique<Entry>();
    e->TreeScore = computeTreeScore(node.get());
    e->ListOfNodes[nodeName] = true;
    e->tree = std::move(node);
    location_[nodeName] = e->tree.get();
    cache_.push_back(std::move(e));
}

void TreeCache::RemoveNodeFromNodeTreeCache(const std::string &nodeName) {
    removeNodeFromCache(nodeName, location(nodeName));
    location_.erase(nodeName);
}

const SortedTreeNode *TreeCache::findBestTreeInCache(int num) const {          // gpu.go:232-245
    const SortedTreeNode *best = nullptr;
    double bestScore = 0.0;
    for (const auto &e : cache_) {
        if (e->tree->Val < num) continue;
        if (e->TreeScore > bestScore ||
            (best && e->TreeScore == bestScore && compareShape(e->tree.get(), best) < 0)) {
            best = e->tree.get();
            bestScore = e->TreeScore;
        }
    }
    return best;
}

int64_t NvidiaGPUScheduler::PodGPUCount(const types::PodInfo &podInfo) {       // gpu.go:295-303
    int64_t n = 0;
    for (const auto &c : podInfo.RunningContainers) n += getOr0(c.second.Requests, ResourceGPU);
    for (const auto &c : podInfo.InitContainers) n = std::max(n, getOr0(c.second.Requests, ResourceGPU));
    return n;
}

bool ConvertToBestGPURequests(const TreeCache &cache, types::PodInfo &podInfo) {   // gpu.go:294-324
    const int64_t numGPUs = NvidiaGPUScheduler::PodGPUCount(podInfo);
    const SortedTreeNode *best = cache.findBestTreeInCache((int)numGPUs);
    if (!best) return false;
    for (auto &c : podInfo.RunningContainers) translateToTree(best, &c.second);    // sorted names
    for (auto &c : podInfo.InitContainers) translateToTree(best, &c.second);
    return true;
}

std::string TranslatePodGPUResources(const TreeCache &cache, const types::NodeInfo &nodeInfo, types::PodInfo &podInfo,
                                     bool *found) {                             // gpu.go:94-127
    for (auto &c : podInfo.InitContainers) SetGPUReqs(c.second);
    for (auto &c : podInfo.RunningContainers) SetGPUReqs(c.second);
    auto it = podInfo.Requests.find(GPUTopologyGeneration);
    const bool ok = it != podInfo.Requests.end();
    const int64_t req = ok ? it->second : 0;
    *found = true;
    if (!ok || req == 1) {
        *found = ConvertToBestGPURequests(cache, podInfo);
        if (*found) return "";
    }
    if (!*found || req == 0) {
        for (auto &c : podInfo.InitContainers)
            c.second.DevRequests = TranslateGPUResources(getOr0(c.second.Requests, ResourceGPU), nodeInfo.Allocatable, c.second.DevRequests);
        for (auto &c : podInfo.RunningContainers)
            c.second.DevRequests = TranslateGPUResources(getOr0(c.second.Requests, ResourceGPU), nodeInfo.Allocatable, c.second.DevRequests);
        *found = true;
        return "";
    }
    *found = false;
    return "Invalid topology generation request";
}

// ---- NvidiaGPUScheduler -----------------------------------------------------------------
namespace {
// Link levels a 2-level group hierarchy implies (the reference collapses the NVML matrix to
// exactly this before it reaches the scheduler: nvidia_gpu_manager.go:178-180): same gpugrp0
// -> the best level of {6,5,4}; same gpugrp1 -> the best of the rest; otherwise SYSTEM.
constexpr int32_t kLevelSameGrp0 = 5, kLevelSameGrp1 = 3, kLevelCross = 1;

struct GpuSlot {
    std::string grp1, grp0, id, name;
};

// "resource/group/gpugrp1/<a>/gpugrp0/<b>/gpu/<id>/cards" keys -> slots in sorted-key order
std::vector<GpuSlot> parseGpuSlots(const types::ResourceList &alloc) {
    static const std::regex rx(std::string(types::DeviceGroupPrefix) + "/(gpugrp1/(.*?)/gpugrp0/(.*?)/gpu/(.*?))/cards");
    std::vector<GpuSlot> slots;
    std::smatch m;
    for (const auto &kv : alloc)
        if (std::regex_search(kv.first, m, rx) && kv.second > 0) slots.push_back({m[2].str(), m[3].str(), m[4].str(), m[1].str()});
    return slots;
}
}  // namespace

NvidiaGPUScheduler::NvidiaGPUScheduler(const std::vector<int> &devices, bool groupSchedulerMode)
    : groupSchedulerMode_(groupSchedulerMode) {
    if (devices.empty()) return;
    if (kgpu_create(devices.data(), (int)devices.size(), &handle_) != KGPU_OK) {
        lastError_ = kgpu_last_error(nullptr);
        handle_ = nullptr;
    }
}

NvidiaGPUScheduler::~NvidiaGPUScheduler() {
    if (handle_) kgpu_destroy(handle_);
}

const NvidiaGPUScheduler::NodeRecord *NvidiaGPUScheduler::node(const std::string &nodeName) const {
    auto it = nodes_.find(nodeName);
    return it == nodes_.end() ? nullptr : &it->second;
}

void NvidiaGPUScheduler::AddNode(const std::string &nodeName, types::NodeInfo *nodeInfo) {   // gpu_scheduler.go:21-28
    types::ResourceList probe;
    probe[std::string(types::DeviceGroupPrefix) + "/gpugrp1/A/gpugrp0/B/gpu/GPU0/cards"] = 1;
    nodeInfo->Allocatable = TranslateGPUResources(getOr0(nodeInfo->KubeAlloc, ResourceGPU), probe, nodeInfo->Allocatable);
    cache_.AddResourcesToNodeTreeCache(nodeName, nodeInfo->Allocatable);

    // device-side record: up to 8 GPU slots in sorted-name order, matrix from the groups
    NodeRecord &rec = nodes_[nodeName];
    const bool fresh = rec.index < 0;
    if (fresh) {
        rec.name = nodeName;
        rec.index = (int64_t)indexToName_.size();
        indexToName_.push_back(nodeName);
    }
    rec.removed = false;
    infoToName_[nodeInfo] = nodeName;
    const std::vector<GpuSlot> slots = parseGpuSlots(nodeInfo->Allocatable);
    rec.nGpus = (int)std::min<size_t>(slots.size(), KGPU_MAX_GPUS_PER_NODE);
    rec.gpuNames.clear();
    for (int i = 0; i < rec.nGpus; i++) rec.gpuNames.push_back(slots[(size_t)i].name);
    rec.hasMem = false;
    for (int i = 0; i < 8; i++) rec.memMiB[i] = 0;
    for (int i = 0; i < rec.nGpus; i++) {                   // "<name>/memory" next to "<name>/cards" (bytes)
        auto m = nodeInfo->Allocatable.find(std::string(types::DeviceGroupPrefix) + "/" + rec.gpuNames[(size_t)i] + "/memory");
        if (m != nodeInfo->Allocatable.end() && m->second > 0) {
            rec.memMiB[i] = (int32_t)std::min<int64_t>(m->second >> 20, std::numeric_limits<int32_t>::max());
            rec.hasMem = true;
        }
    }
    rec.presentMask = rec.nGpus >= 8 ? 0xFFu : ((1u << rec.nGpus) - 1u);
    rec.usedMask &= rec.presentMask;
    if (!rec.explicitTopo) {
        std::fill(rec.topo, rec.topo + 64, 0);
        for (int i = 0; i < rec.nGpus; i++)
            for (int j = 0; j < rec.nGpus; j++) {
                if (i == j) continue;
                const GpuSlot &a = slots[(size_t)i], &b = slots[(size_t)j];
                rec.topo[i * 8 + j] = (a.grp1 == b.grp1 && a.grp0 == b.grp0) ? kLevelSameGrp0
                                      : (a.grp1 == b.grp1)                    ? kLevelSameGrp1
                                                                              : kLevelCross;
            }
    }
    if (fresh) dirty_ = true; else changed_.push_back(nodeName);
    holdersChanged_.insert(nodeName);
}

void NvidiaGPUScheduler::RemoveNode(const std::string &nodeName) {              // gpu_scheduler.go:30-32
    cache_.RemoveNodeFromNodeTreeCache(nodeName);
    auto it = nodes_.find(nodeName);
    if (it != nodes_.end()) {
        it->second.removed = true;
        changed_.push_back(nodeName);
        holdersChanged_.insert(nodeName);
    }
}

std::string NvidiaGPUScheduler::SetNodeTopology(const std::string &nodeName, const int32_t topo[64]) {
    auto it = nodes_.find(nodeName);
    if (it == nodes_.end()) return lastError_ = "SetNodeTopology: unknown node " + nodeName;
    for (int i = 0; i < 64; i++)
        if (topo[i] < 0 || topo[i] >= KGPU_NUM_LEVELS) return lastError_ = "SetNodeTopology: link level outside 0..15";
    std::copy(topo, topo + 64, it->second.topo);
    it->second.explicitTopo = true;
    changed_.push_back(nodeName);
    return "";
}

std::string NvidiaGPUScheduler::AddNodeFromGpusInfo(const std::string &nodeName, const std::string &gpusInfoJSON,
                                                    bool useNVML, types::NodeInfo *nodeInfo) {
    nvgputypes::GpusInfo info;
    std::string err = nvgputypes::ParseGpusInfo(gpusInfoJSON, &info);
    if (!err.empty()) return lastError_ = err;
    if (info.Gpus.size() > KGPU_MAX_GPUS_PER_NODE) return lastError_ = "AddNodeFromGpusInfo: more than 8 GPUs on " + nodeName;
    nvidia::DiscoverTopology(&info, useNVML);
    *nodeInfo = types::NodeInfo();
    nodeInfo->Name = nodeName;
    nvidia::UpdateNodeInfo(info, nodeInfo);
    AddNode(nodeName, nodeInfo);
    // slot i of the node record = i-th advertised name in sorted order; map it back to the GPU
    const NodeRecord *rec = node(nodeName);
    const std::vector<int32_t> links = nvidia::LinkMatrix(info);
    const size_t n = info.Gpus.size();
    std::vector<size_t> gpuOfSlot;
    for (const std::string &slotName : rec->gpuNames)
        for (size_t g = 0; g < n; g++)
            if (info.Gpus[g].Name == slotName) { gpuOfSlot.push_back(g); break; }
    if (gpuOfSlot.size() != rec->gpuNames.size()) return lastError_ = "AddNodeFromGpusInfo: advertised names do not map back to GPUs";
    int32_t topo[64] = {0};
    for (size_t i = 0; i < gpuOfSlot.size(); i++)
        for (size_t j = 0; j < gpuOfSlot.size(); j++)
            if (i != j) {
                const int32_t l = links[gpuOfSlot[i] * n + gpuOfSlot[j]];
                if (l < 0 || l >= KGPU_NUM_LEVELS) return lastError_ = "AddNodeFromGpusInfo: link level outside 0..15";
                topo[i * 8 + j] = l;
            }
    return SetNodeTopology(nodeName, topo);
}

std::string NvidiaGPUScheduler::SetNodeDomain(const std::string &nodeName, const std::string &domainName) {
    return SetNodeDomains(nodeName, {domainName});
}

std::string NvidiaGPUScheduler::SetNodeDomains(const std::string &nodeName, const std::vector<std::string> &names) {
    auto it = nodes_.find(nodeName);
    if (it == nodes_.end()) return lastError_ = "SetNodeDomain: unknown node " + nodeName;
    if ((int)names.size() > KGPU_MAX_DOMAIN_LEVELS)
        return lastError_ = "SetNodeDomains: " + std::to_string(names.size()) + " levels, at most " + std::to_string(KGPU_MAX_DOMAIN_LEVELS);
    if (it->second.domains != names) domainsDirty_ = true;
    it->second.domains = names;
    return "";
}

// The domain table on the device, if a domain or the node array changed since the last push: per level, names -> ids
// 0, 1, ... in sorted order, -1 for nodes without one; as many levels as the longest list.
std::string NvidiaGPUScheduler::pushDomains() {
    if (!domainsDirty_) return "";
    const size_t n = indexToName_.size();
    size_t levels = 1;
    for (const std::string &name : indexToName_) levels = std::max(levels, nodes_[name].domains.size());
    std::vector<int32_t> domain(levels * n, -1);
    for (size_t l = 0; l < levels; l++) {
        std::map<std::string, int32_t> ids;
        for (const std::string &name : indexToName_) {
            const std::vector<std::string> &d = nodes_[name].domains;
            if (l < d.size() && !d[l].empty()) ids.emplace(d[l], 0);
        }
        int32_t next = 0;
        for (auto &kv : ids) kv.second = next++;
        for (size_t i = 0; i < n; i++) {
            const std::vector<std::string> &d = nodes_[indexToName_[i]].domains;
            if (l < d.size() && !d[l].empty()) domain[l * n + i] = ids[d[l]];
        }
    }
    if (kgpu_upload_domain_levels(handle_, domain.data(), (int)levels, (int64_t)n) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
    domainsDirty_ = false;
    return "";
}

// Push the host-side node array to the device(s) if it changed since the last launch.
std::string NvidiaGPUScheduler::flushNodes() {
    if (!handle_) return lastError_ = "no CUDA device: the kgpu scorer has no CPU path (" + lastError_ + ")";
    if (!dirty_) {
        // only existing nodes changed: one kgpu_update_node each (256-byte copy + a refresh of that node's records)
        // instead of re-uploading the cluster
        for (const std::string &name : changed_) {
            const NodeRecord &rec = nodes_[name];
            const int32_t fm = rec.removed ? 0 : (int32_t)(rec.presentMask & ~rec.usedMask);
            if (kgpu_update_node(handle_, rec.index, rec.topo, fm) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
            if (rec.hasMem) {
                int32_t mem[8];
                for (int g = 0; g < 8; g++) mem[g] = g < rec.nGpus ? rec.memMiB[g] : 0;
                if (kgpu_update_gpu_memory(handle_, rec.index, mem) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
            }
        }
        changed_.clear();
        return "";
    }
    changed_.clear();
    const size_t n = indexToName_.size();
    std::vector<int32_t> topo(n * 64), freeMask(n);
    for (size_t i = 0; i < n; i++) {
        const NodeRecord &rec = nodes_[indexToName_[i]];
        std::copy(rec.topo, rec.topo + 64, topo.begin() + (std::ptrdiff_t)(i * 64));
        freeMask[i] = rec.removed ? 0 : (int32_t)(rec.presentMask & ~rec.usedMask);
    }
    if (kgpu_upload_nodes(handle_, topo.data(), freeMask.data(), (int64_t)n, 0) != KGPU_OK)
        return lastError_ = kgpu_last_error(handle_);
    bool anyMem = false;
    std::vector<int32_t> mem(n * 8, std::numeric_limits<int32_t>::max());     // unknown = unconstrained
    for (size_t i = 0; i < n; i++) {
        const NodeRecord &rec = nodes_[indexToName_[i]];
        if (!rec.hasMem) continue;
        anyMem = true;
        for (int g = 0; g < 8; g++) mem[i * 8 + (size_t)g] = g < rec.nGpus ? rec.memMiB[g] : 0;
    }
    if (anyMem && kgpu_upload_gpu_memory(handle_, mem.data(), (int64_t)n) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
    dirty_ = false;
    holdersReset_ = true;                                // kgpu_upload_nodes reset the holder table
    domainsDirty_ = true;                                // and the domain table
    return "";
}

std::string NvidiaGPUScheduler::ScoreBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out) {
    return runBatch(pods, out, BatchMode::Snapshot);
}

std::string NvidiaGPUScheduler::PlaceBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out) {
    return runBatch(pods, out, BatchMode::Sequential);
}

std::string NvidiaGPUScheduler::ProposeBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out) {
    return runBatch(pods, out, BatchMode::DryRun);
}

namespace {
int32_t minMemOf(const types::PodInfo &pod) {
    const int64_t need = getOr0(pod.Requests, GPUMinMemoryMiB);
    return (int32_t)std::max<int64_t>(0, std::min<int64_t>(need, std::numeric_limits<int32_t>::max()));
}
int levelOf(const types::PodInfo &pod) {
    return (int)std::max<int64_t>(0, std::min<int64_t>(getOr0(pod.Requests, GPUPriorityLevel), 15));
}
}  // namespace

std::string NvidiaGPUScheduler::PreemptBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                             std::vector<std::vector<std::string>> *victims) {
    return runBatch(pods, out, BatchMode::Preempt, victims);
}

std::string NvidiaGPUScheduler::PlanPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                               std::vector<std::vector<std::string>> *victims) {
    return runBatch(pods, out, BatchMode::PreemptPlan, victims);
}

std::string NvidiaGPUScheduler::PlanGangPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                                   std::vector<std::vector<std::string>> *victims) {
    return runBatch(pods, out, BatchMode::PreemptGangPlan, victims);
}

std::string NvidiaGPUScheduler::PlanGangDomainPreemption(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                                         std::vector<std::vector<std::string>> *victims) {
    return runBatch(pods, out, BatchMode::PreemptGangDomainPlan, victims);
}

// Holder rows from the committed placements: on each node the pods holding GPUs, in name order, are owners 0, 1, ...;
// a GPU gets level << 3 | owner of the pod that holds it, -1 if no committed placement accounts for it.  Pushed for the
// nodes changed since the last push (kgpu_set_holders), or all of them after a re-upload reset the table.
std::string NvidiaGPUScheduler::pushHolders() {
    std::vector<std::string> names;
    if (holdersReset_) {
        names = indexToName_;
    } else {
        names.assign(holdersChanged_.begin(), holdersChanged_.end());
    }
    std::map<std::string, std::vector<std::pair<std::string, const Placement *>>> held;   // node -> (pod, placement)
    for (const auto &kv : lastPlacement_)                   // std::map: pods in name order
        if (kv.second.fits && kv.second.committed && kv.second.gpuMask) held[kv.second.nodeName].emplace_back(kv.first, &kv.second);
    std::vector<int64_t> idx;
    std::vector<int32_t> rows;
    for (const std::string &name : names) {
        auto it = nodes_.find(name);
        if (it == nodes_.end()) continue;
        NodeRecord &rec = it->second;
        int32_t row[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
        rec.owners.clear();
        if (!rec.removed) {
            for (const auto &hp : held[name]) {
                if (rec.owners.size() == 8) break;
                const uint32_t mask = hp.second->gpuMask & rec.usedMask;
                if (!mask) continue;
                const int32_t o = (int32_t)rec.owners.size();
                rec.owners.push_back(hp.first);
                for (int g = 0; g < 8; g++)
                    if ((mask >> g) & 1u) row[g] = (int32_t)hp.second->level << 3 | o;
            }
        }
        idx.push_back(rec.index);
        rows.insert(rows.end(), row, row + 8);
    }
    if (!idx.empty() && kgpu_set_holders(handle_, idx.data(), rows.data(), (int64_t)idx.size()) != KGPU_OK)
        return lastError_ = kgpu_last_error(handle_);
    holdersChanged_.clear();
    holdersReset_ = false;
    return "";
}

std::string NvidiaGPUScheduler::runBatch(const std::vector<const types::PodInfo *> &pods, std::vector<Placement> *out,
                                         BatchMode mode, std::vector<std::vector<std::string>> *victims) {
    std::string err = flushNodes();
    if (!err.empty()) return err;
    const size_t P = pods.size();
    // Gangs (sequential modes and gang plans only): the device takes a gang as one run of consecutive pods with an int32 id, so the
    // ids are renumbered 1, 2, ... in order of first appearance (no truncation can merge two gangs) and each member
    // moves up to its gang's first member.  order[i] = the caller's index of the pod at device position i.
    std::vector<size_t> order(P);
    std::vector<int32_t> gang, gangDomain, gangLevel;   // in device order, empty when no pod asks for a domain / level
    for (size_t p = 0; p < P; p++) order[p] = p;
    const bool placing = mode == BatchMode::Sequential || mode == BatchMode::DryRun;
    if (placing || mode == BatchMode::PreemptGangDomainPlan) {
        std::map<int64_t, int64_t> domainOfGang, levelOfGang;
        for (size_t p = 0; p < P; p++) {
            const int64_t gd = getOr0(pods[p]->Requests, GPUGangDomain), id = getOr0(pods[p]->Requests, GPUGangID);
            const int64_t gl = getOr0(pods[p]->Requests, GPUGangDomainLevel);
            if (gl != 0 && mode == BatchMode::PreemptGangDomainPlan)
                return lastError_ = "pod " + pods[p]->Name + ": " + GPUGangDomainLevel + " is not supported in preemption plans (level 0 only)";
            if (gl != 0 && gd == 0) return lastError_ = "pod " + pods[p]->Name + ": " + GPUGangDomainLevel + " without " + GPUGangDomain;
            if (gl < 0 || gl >= KGPU_MAX_DOMAIN_LEVELS)
                return lastError_ = "pod " + pods[p]->Name + ": " + GPUGangDomainLevel + " must be 0.." + std::to_string(KGPU_MAX_DOMAIN_LEVELS - 1);
            if (id != 0 && !levelOfGang.emplace(id, gl).second && levelOfGang[id] != gl)
                return lastError_ = "pod " + pods[p]->Name + ": the members of gang " + std::to_string(id) + " disagree on " + GPUGangDomainLevel;
            if (gl != 0) gangLevel.assign(P, 0);
            if (gd != 0 && gd != KGPU_GANG_DOMAIN_REQUIRED && gd != KGPU_GANG_DOMAIN_PREFERRED)
                return lastError_ = "pod " + pods[p]->Name + ": " + GPUGangDomain + " must be 1 (required) or 2 (preferred)";
            if (gd != 0 && id == 0) return lastError_ = "pod " + pods[p]->Name + ": " + GPUGangDomain + " without " + GPUGangID;
            if (id != 0 && !domainOfGang.emplace(id, gd).second && domainOfGang[id] != gd)
                return lastError_ = "pod " + pods[p]->Name + ": the members of gang " + std::to_string(id) + " disagree on " + GPUGangDomain;
            if (gd != 0) gangDomain.assign(P, 0);
        }
        err = pushDomains();
        if (!err.empty()) return err;
    }
    if (placing || mode == BatchMode::PreemptGangPlan || mode == BatchMode::PreemptGangDomainPlan) {
        std::map<int64_t, int32_t> dense;
        std::vector<std::vector<size_t>> members;
        std::vector<int32_t> gangOf(P, 0);
        for (size_t p = 0; p < P; p++) {
            const int64_t id = getOr0(pods[p]->Requests, GPUGangID);
            if (id == 0) continue;
            const auto it = dense.emplace(id, (int32_t)dense.size() + 1).first;
            if ((size_t)it->second > members.size()) members.emplace_back();
            gangOf[p] = it->second;
            members[(size_t)it->second - 1].push_back(p);
        }
        if (!members.empty()) {
            order.clear();
            gang.reserve(P);
            std::vector<bool> done(members.size(), false);
            for (size_t p = 0; p < P; p++) {
                const int32_t g = gangOf[p];
                if (g == 0) {
                    order.push_back(p);
                    gang.push_back(0);
                } else if (!done[(size_t)g - 1]) {
                    done[(size_t)g - 1] = true;
                    for (size_t m : members[(size_t)g - 1]) {
                        order.push_back(m);
                        gang.push_back(g);
                    }
                }
            }
        }
    }
    std::vector<int32_t> req(P * 4, 0);
    for (size_t i = 0; i < P; i++) {
        const size_t p = order[i];
        if (!gangDomain.empty()) gangDomain[i] = (int32_t)getOr0(pods[p]->Requests, GPUGangDomain);
        if (!gangLevel.empty()) gangLevel[i] = (int32_t)getOr0(pods[p]->Requests, GPUGangDomainLevel);
        types::PodInfo copy = *pods[p];                    // SetGPUReqs mutates; keep the caller's pod intact
        for (auto &c : copy.InitContainers) SetGPUReqs(c.second);
        for (auto &c : copy.RunningContainers) SetGPUReqs(c.second);
        const int64_t k = PodGPUCount(copy);
        req[i * 4 + 0] = k > 8 ? 9 : (int32_t)k;           // > 8 GPUs never fits one node
        req[i * 4 + 1] = (int32_t)p;
        req[i * 4 + 3] = minMemOf(*pods[p]);
    }
    std::vector<uint64_t> dev(P, KGPU_NO_FIT);
    std::vector<uint32_t> owners(P, 0);
    std::vector<int32_t> lvl(P, 0);
    const bool preempt = mode == BatchMode::Preempt || mode == BatchMode::PreemptPlan || mode == BatchMode::PreemptGangPlan ||
                         mode == BatchMode::PreemptGangDomainPlan;
    if (preempt) {
        for (size_t i = 0; i < P; i++) lvl[i] = levelOf(*pods[order[i]]);
        err = pushHolders();
        if (!err.empty()) return err;
    }
    const int rc = mode == BatchMode::Preempt  ? kgpu_preempt_batch(handle_, req.data(), lvl.data(), (int64_t)P, dev.data(), owners.data())
                   : mode == BatchMode::PreemptPlan ? kgpu_preempt_plan(handle_, req.data(), lvl.data(), (int64_t)P, dev.data(), owners.data())
                   : mode == BatchMode::PreemptGangPlan
                       ? kgpu_preempt_plan_gang(handle_, req.data(), lvl.data(), gang.empty() ? nullptr : gang.data(), (int64_t)P,
                                                dev.data(), owners.data())
                   : mode == BatchMode::PreemptGangDomainPlan
                       ? kgpu_preempt_plan_gang_domain(handle_, req.data(), lvl.data(), gang.empty() ? nullptr : gang.data(),
                                                       gangDomain.empty() ? nullptr : gangDomain.data(), (int64_t)P, dev.data(),
                                                       owners.data())
                   : mode == BatchMode::Snapshot ? kgpu_score_batch(handle_, req.data(), (int64_t)P, dev.data())
                                               : kgpu_place_batch_gang_levels(handle_, req.data(), gang.empty() ? nullptr : gang.data(),
                                                                              gangDomain.empty() ? nullptr : gangDomain.data(),
                                                                              gangLevel.empty() ? nullptr : gangLevel.data(), (int64_t)P,
                                                                              dev.data(), mode == BatchMode::DryRun ? KGPU_PLACE_DRY_RUN : 0);
    if (rc != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
    std::vector<uint64_t> keys(P, KGPU_NO_FIT);           // back in the caller's order
    std::vector<uint32_t> vic(P, 0);
    for (size_t i = 0; i < P; i++) {
        keys[order[i]] = dev[i];
        vic[order[i]] = owners[i];
    }
    out->assign(P, Placement());
    if (victims) victims->assign(P, {});
    for (size_t p = 0; p < P; p++) {
        Placement &pl = (*out)[p];
        pl.key = keys[p];
        pl.level = levelOf(*pods[p]);
        if (keys[p] != KGPU_NO_FIT) {
            pl.fits = true;
            pl.cost = KGPU_KEY_COST(keys[p]);
            pl.gpuMask = KGPU_KEY_MASK(keys[p]);
            pl.nodeName = indexToName_[KGPU_KEY_NODE(keys[p])];
            if (mode == BatchMode::Sequential) {            // the device already took them: TakePodResources is a no-op
                nodes_[pl.nodeName].usedMask |= pl.gpuMask;
                pl.committed = true;
                holdersChanged_.insert(pl.nodeName);
            }
            if (preempt) {
                const NodeRecord &rec = nodes_[pl.nodeName];
                for (int o = 0; o < 8; o++)
                    if (((vic[p] >> o) & 1u) && (size_t)o < rec.owners.size()) (*victims)[p].push_back(rec.owners[(size_t)o]);
            }
        }
        if (preempt) continue;                               // a proposal that needs evictions first: not remembered
        if (!pods[p]->Name.empty()) lastPlacement_[pods[p]->Name] = pl;
    }
    return "";
}

// Which registered node is this?  The reference passes only the NodeInfo: its Name, else the pointer AddNode saw.
const NvidiaGPUScheduler::NodeRecord *NvidiaGPUScheduler::recordOf(const types::NodeInfo *nodeInfo) const {
    const NodeRecord *rec = nullptr;
    if (!nodeInfo->Name.empty()) rec = node(nodeInfo->Name);
    if (!rec) {
        auto byPtr = infoToName_.find(nodeInfo);
        if (byPtr != infoToName_.end()) rec = node(byPtr->second);
    }
    return (rec && !rec->removed) ? rec : nullptr;
}

// (cost<<8 | mask) of this node for k GPUs: the handle's (node, k) fit table (a host read, no launch) unless the
// pod carries a memory requirement (one packed query launch).
std::string NvidiaGPUScheduler::scoreOne(const NodeRecord &rec, int k, int32_t minMemMiB, uint32_t *nodeKey) {
    std::string err = flushNodes();
    if (!err.empty()) return err;
    const int32_t kk = k > 8 ? 9 : k;
    if (minMemMiB <= 0) {
        if (kgpu_fit_lookup(handle_, rec.index, kk, nodeKey) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
        return "";
    }
    const int64_t idx = rec.index;
    if (kgpu_score_pairs(handle_, &idx, &kk, &minMemMiB, 1, nodeKey) != KGPU_OK) return lastError_ = kgpu_last_error(handle_);
    return "";
}

// gpu_scheduler.go:34-44.  fits / reasons as the reference, PLUS the device's verdict for this node's current free
// GPUs; `score` is the new part: 1 / (1 + link cost of the cheapest k-subset of THIS node's free GPUs), 0 when the
// GPUs do not fit.  Higher is better, 1.0 = all requested GPUs on zero-cost (NVLink) links.  The fits decision
// does not depend on whether the caller asked for a score, and a device error is a "does not fit" with a reason
// (the reference collapses errors to false as well, gpu_scheduler.go:35-42), never a silent "fits, score 0".
bool NvidiaGPUScheduler::PodFitsDevice(types::NodeInfo *nodeInfo, types::PodInfo *podInfo, bool fillAllocateFrom,
                                       std::vector<kubedevice::devicescheduler::PredicateFailureReason> *reasons,
                                       double *score) {
    if (reasons) reasons->clear();
    if (score) *score = 0.0;
    bool found = false;
    const std::string err = TranslatePodGPUResources(cache_, *nodeInfo, *podInfo, &found);
    if (!err.empty() || !found) return false;
    if (!handle_) return true;                                // host-only mode: the reference's answer
    const NodeRecord *rec = recordOf(nodeInfo);
    if (!rec) return true;                                    // a node AddNode never saw: the reference's answer, score 0.0
    uint32_t nk = UINT32_MAX;
    const std::string derr = scoreOne(*rec, (int)PodGPUCount(*podInfo), minMemOf(*podInfo), &nk);
    if (!derr.empty()) {
        if (reasons) reasons->push_back({"kgpu: " + derr});
        return false;
    }
    if (nk == UINT32_MAX) {                                   // a feasible shape exists in the cache, but not on this node now
        if (reasons) reasons->push_back({"kgpu: not enough free GPUs on " + rec->name});
        return false;
    }
    if (score) *score = 1.0 / (1.0 + (double)(nk >> 8));
    if (fillAllocateFrom && !groupSchedulerMode_ && !podInfo->Name.empty()) {
        Placement pl;                                         // remember the per-node placement for PodAllocate
        pl.fits = true;
        pl.cost = nk >> 8;
        pl.gpuMask = nk & 0xFFu;
        pl.nodeName = rec->name;
        pl.level = levelOf(*podInfo);
        pl.key = ((uint64_t)pl.cost << 40) | ((uint64_t)rec->index << 8) | pl.gpuMask;
        lastPlacement_[podInfo->Name] = pl;
    }
    return true;
}

// gpu_scheduler.go:46-55 plus SURVEY.md 8(f) rank 1: expand (node, mask) into AllocateFrom: request name -> the
// node's own resource name, which the node agent's Allocate regex (nvidia_gpu_manager.go:225-241) turns into
// NVIDIA_VISIBLE_DEVICES.  The placement is the one ScoreBatch / ProposeBatch / PlaceBatch / PodFitsDevice
// recorded for this pod ON THIS NODE; without one it is computed now for this node.  Containers take GPUs in
// sorted-name order, lowest slot first.  groupSchedulerMode: the reference's behaviour only (DevRequests).
std::string NvidiaGPUScheduler::PodAllocate(types::NodeInfo *nodeInfo, types::PodInfo *podInfo) {
    bool found = false;
    const std::string err = TranslatePodGPUResources(cache_, *nodeInfo, *podInfo, &found);
    if (!err.empty()) return err;
    if (!found) return "TranslatePodGPUResources fails as no translation is found";
    if (groupSchedulerMode_ || !handle_) return "";
    const NodeRecord *here = recordOf(nodeInfo);
    Placement pl;
    auto it = podInfo->Name.empty() ? lastPlacement_.end() : lastPlacement_.find(podInfo->Name);
    if (it != lastPlacement_.end() && it->second.fits && (!here || here->name == it->second.nodeName)) {
        pl = it->second;
    } else if (here) {                                        // no placement recorded for this node: ask the device now
        uint32_t nk = UINT32_MAX;
        const std::string derr = scoreOne(*here, (int)PodGPUCount(*podInfo), minMemOf(*podInfo), &nk);
        if (!derr.empty()) return derr;
        if (nk == UINT32_MAX) return "PodAllocate: not enough free GPUs on " + here->name;
        pl.fits = true;
        pl.cost = nk >> 8;
        pl.gpuMask = nk & 0xFFu;
        pl.nodeName = here->name;
        pl.level = levelOf(*podInfo);
        pl.key = ((uint64_t)pl.cost << 40) | ((uint64_t)here->index << 8) | pl.gpuMask;
        if (!podInfo->Name.empty()) lastPlacement_[podInfo->Name] = pl;
    } else {
        return "";
    }
    const NodeRecord *rec = node(pl.nodeName);
    if (!rec) return "";
    std::vector<int> slotsLeft;
    for (int i = 0; i < 8; i++)
        if ((pl.gpuMask >> i) & 1u) slotsLeft.push_back(i);
    size_t next = 0;
    auto fill = [&](types::ContainerInfo &cont, size_t *cursor) {
        cont.AllocateFrom.clear();
        for (const auto &kv : cont.DevRequests) {
            if (kv.first.find("/gpu/") == std::string::npos || kv.first.size() < 6 ||
                kv.first.compare(kv.first.size() - 6, 6, "/cards") != 0)
                continue;
            if (*cursor >= slotsLeft.size()) break;
            cont.AllocateFrom[kv.first] = std::string(types::DeviceGroupPrefix) + "/" + rec->gpuNames[(size_t)slotsLeft[*cursor]] + "/cards";
            (*cursor)++;
        }
    };
    for (auto &c : podInfo->RunningContainers) fill(c.second, &next);
    for (auto &c : podInfo->InitContainers) {                  // init containers run before, reuse the same GPUs
        size_t cur = 0;
        fill(c.second, &cur);
    }
    return "";
}

std::string NvidiaGPUScheduler::pushMask(NodeRecord &rec) {
    if (!handle_ || dirty_) return "";                        // host-only, or a re-upload is pending anyway
    for (const std::string &c : changed_)
        if (c == rec.name) return "";                         // kgpu_update_node will carry the mask
    if (kgpu_set_free_mask(handle_, rec.index, (int32_t)(rec.removed ? 0 : (rec.presentMask & ~rec.usedMask))) != KGPU_OK)
        return lastError_ = kgpu_last_error(handle_);
    return "";
}

// gpu_scheduler.go:57-63 are no-ops in the reference (the core tracks usage).  Here they keep the device-side free
// masks current (SURVEY.md 8(f) rank 2).  Take is idempotent: a placement PlaceBatch already committed on the
// device, or one taken before, succeeds without touching anything (callers of the reference never see an error
// from these methods); GPUs that are in use by ANOTHER pod are an error -- the caller must re-score that pod.
std::string NvidiaGPUScheduler::TakePodResources(types::NodeInfo * /*nodeInfo*/, types::PodInfo *podInfo) {
    auto it = lastPlacement_.find(podInfo->Name);
    if (podInfo->Name.empty() || it == lastPlacement_.end() || !it->second.fits) return "";
    if (it->second.committed) return "";
    auto n = nodes_.find(it->second.nodeName);
    if (n == nodes_.end()) return "";
    if (n->second.usedMask & it->second.gpuMask)
        return lastError_ = "TakePodResources: GPUs of pod " + podInfo->Name + " already in use on " + n->first + " (score the pod again)";
    n->second.usedMask |= it->second.gpuMask;
    it->second.committed = true;
    holdersChanged_.insert(n->first);
    return pushMask(n->second);
}

std::string NvidiaGPUScheduler::ReturnPodResources(types::NodeInfo * /*nodeInfo*/, types::PodInfo *podInfo) {
    auto it = lastPlacement_.find(podInfo->Name);
    if (podInfo->Name.empty() || it == lastPlacement_.end() || !it->second.fits) return "";
    auto n = nodes_.find(it->second.nodeName);
    if (n == nodes_.end() || !it->second.committed) {          // never taken: just forget the proposal
        lastPlacement_.erase(it);
        return "";
    }
    n->second.usedMask &= ~it->second.gpuMask;
    lastPlacement_.erase(it);
    holdersChanged_.insert(n->first);
    return pushMask(n->second);
}

std::unique_ptr<NvidiaGPUScheduler> CreateDeviceSchedulerPlugin(std::string *err) {
    auto s = std::make_unique<NvidiaGPUScheduler>(std::vector<int>{0});
    if (!s->hasDevice()) {
        if (err) *err = s->LastError();
        return nullptr;
    }
    return s;
}

}  // namespace gpuschedulerplugin
