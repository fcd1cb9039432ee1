// sched_cli.cc -- line-protocol driver for the C++ DeviceScheduler mirror.
//
// Stands in for the external KubeDevice core (absent from the reference tree) so the host
// layer can be driven from tests: tests/test_host_scheduler.py feeds the same script to this
// binary and to the Python oracle and compares the transcripts.
//
//   kgpu_sched_cli [--no-device]  < script  > transcript
//
// Commands (space separated; resource names never contain spaces):
//   addnode NAME KUBEALLOC [key=val ...]        AddNode with Allocatable = {key: val}
//   rmnode NAME                                 RemoveNode
//   topo NAME v0 .. v63                         SetNodeTopology (extension)
//   domain NODE [NAME0 [NAME1 ...]]             SetNodeDomains (extension): the node's network domain per level (level 0
//                                               the finest), none without a NAME; "-" = none at that level
//   pod NAME [topogen=V] [minmem=MiB] [gang=ID] [gangdomain=required|preferred] [gangdomainlevel=R] [priority=L]
//       {run|init CNAME req=N [kube=N] [dev:key=val ...]}...
//   fits NODE POD                               PodFitsDevice  -> fits/score + rewritten requests
//   allocate NODE POD                           PodAllocate    -> error text + AllocateFrom
//   take POD | return POD                       TakePodResources / ReturnPodResources
//   scorebatch POD...                           ScoreBatch (GPU)
//   placebatch POD...                           PlaceBatch (GPU, sequential, takes the GPUs)
//   proposebatch POD...                         ProposeBatch (GPU, sequential on a scratch copy, takes nothing)
//   preemptbatch POD...                         PreemptBatch (GPU): placements when lower-priority pods may be evicted
//   preemptplan POD...                          PlanPreemption (GPU): the same in order, no victim or GPU named twice
//   preemptgangplan POD...                      PlanGangPreemption (GPU): preemptplan with gangs, all members or none
//   preemptdomainplan POD...                    PlanGangDomainPreemption (GPU): preemptgangplan with gang domains
//   addjson NAME FILE [nvml]                    AddNodeFromGpusInfo (node agent JSON), dumps names + matrix
//   visible POD                                 NVIDIA_VISIBLE_DEVICES per container (node agent Allocate)
//   cache                                       dump the tree cache
//   best K                                      findBestTreeInCache(K)
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <iostream>
#include <sstream>

#include <fstream>

#include "device_scheduler.h"
#include "gpus_info.h"

using namespace gpuschedulerplugin;
namespace types = kubedevice::types;

namespace {

std::map<std::string, types::NodeInfo> g_nodes;
std::map<std::string, types::PodInfo> g_pods;

bool splitKV(const std::string &tok, std::string *k, long long *v) {
    const size_t eq = tok.rfind('=');
    if (eq == std::string::npos) return false;
    *k = tok.substr(0, eq);
    *v = atoll(tok.c_str() + eq + 1);
    return true;
}

void dumpPod(const types::PodInfo &pod) {
    auto dump = [](const char *kind, const std::map<std::string, types::ContainerInfo> &cs) {
        for (const auto &c : cs) {
            printf("  %s %s req=%lld\n", kind, c.first.c_str(),
                   (long long)(c.second.Requests.count(gpuplugintypes::ResourceGPU) ? c.second.Requests.at(gpuplugintypes::ResourceGPU) : -1));
            for (const auto &kv : c.second.DevRequests) printf("    dev %s=%lld\n", kv.first.c_str(), (long long)kv.second);
            for (const auto &kv : c.second.AllocateFrom) printf("    from %s -> %s\n", kv.first.c_str(), kv.second.c_str());
        }
    };
    dump("run", pod.RunningContainers);
    dump("init", pod.InitContainers);
}

}  // namespace

int main(int argc, char **argv) {
    bool noDevice = false, groupMode = false;
    for (int i = 1; i < argc; i++) {
        if (std::string(argv[i]) == "--no-device") noDevice = true;
        if (std::string(argv[i]) == "--group-scheduler") groupMode = true;      // the reference's contract: see device_scheduler.h
    }
    NvidiaGPUScheduler sched(noDevice ? std::vector<int>{} : std::vector<int>{0}, groupMode);
    if (!noDevice && !sched.hasDevice()) {
        fprintf(stderr, "kgpu_sched_cli: %s\n", sched.LastError().c_str());
        return 2;
    }
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string cmd;
        if (!(in >> cmd) || cmd[0] == '#') continue;
        printf("> %s\n", line.c_str());
        if (cmd == "addnode") {
            std::string name, tok, k;
            long long kube = 0, v = 0;
            in >> name >> kube;
            types::NodeInfo &ni = g_nodes[name];
            ni = types::NodeInfo();
            ni.Name = name;
            ni.KubeAlloc[gpuplugintypes::ResourceGPU] = kube;
            while (in >> tok)
                if (splitKV(tok, &k, &v)) ni.Allocatable[k] = v;
            sched.AddNode(name, &ni);
            for (const auto &kv : ni.Allocatable) printf("  alloc %s=%lld\n", kv.first.c_str(), (long long)kv.second);
        } else if (cmd == "addjson") {
            std::string name, file, mode;
            in >> name >> file >> mode;
            std::ifstream f(file);
            std::stringstream buf;
            buf << f.rdbuf();
            types::NodeInfo &ni = g_nodes[name];
            const std::string err = sched.AddNodeFromGpusInfo(name, buf.str(), mode == "nvml", &ni);
            printf("  err=%s\n", err.c_str());
            for (const auto &kv : ni.Allocatable) printf("  alloc %s=%lld\n", kv.first.c_str(), (long long)kv.second);
            if (const auto *rec = sched.node(name)) {
                for (int i = 0; i < 8; i++) {
                    printf("  topo");
                    for (int j = 0; j < 8; j++) printf(" %d", rec->topo[i * 8 + j]);
                    printf("\n");
                }
            }
        } else if (cmd == "visible") {
            std::string podName;
            in >> podName;
            if (!g_pods.count(podName)) { printf("  unknown pod\n"); continue; }
            for (const auto &c : g_pods[podName].RunningContainers)
                printf("  %s NVIDIA_VISIBLE_DEVICES=%s\n", c.first.c_str(), nvidia::VisibleDevices(c.second).c_str());
        } else if (cmd == "rmnode") {
            std::string name;
            in >> name;
            sched.RemoveNode(name);
        } else if (cmd == "topo") {
            std::string name;
            int32_t t[64];
            in >> name;
            for (int i = 0; i < 64; i++) in >> t[i];
            printf("  err=%s\n", sched.SetNodeTopology(name, t).c_str());
        } else if (cmd == "domain") {
            std::string name, dom;
            std::vector<std::string> names;
            in >> name;
            while (in >> dom) names.push_back(dom == "-" ? "" : dom);
            printf("  err=%s\n", names.size() <= 1 ? sched.SetNodeDomain(name, names.empty() ? "" : names[0]).c_str()
                                                  : sched.SetNodeDomains(name, names).c_str());
        } else if (cmd == "pod") {
            std::string name, tok, k;
            long long v = 0;
            in >> name;
            types::PodInfo &pod = g_pods[name];
            pod = types::PodInfo();
            pod.Name = name;
            types::ContainerInfo *cur = nullptr;
            while (in >> tok) {
                if (tok == "run" || tok == "init") {
                    std::string cname;
                    in >> cname;
                    cur = tok == "run" ? &pod.RunningContainers[cname] : &pod.InitContainers[cname];
                } else if (tok.compare(0, 8, "topogen=") == 0) {
                    pod.Requests[GPUTopologyGeneration] = atoll(tok.c_str() + 8);
                } else if (tok.compare(0, 7, "minmem=") == 0) {
                    pod.Requests[GPUMinMemoryMiB] = atoll(tok.c_str() + 7);
                } else if (tok.compare(0, 5, "gang=") == 0) {
                    pod.Requests[GPUGangID] = atoll(tok.c_str() + 5);
                } else if (tok.compare(0, 11, "gangdomain=") == 0) {
                    const std::string gd = tok.substr(11);
                    pod.Requests[GPUGangDomain] = gd == "required" ? 1
                                                  : gd == "preferred" ? 2
                                                                      : atoll(gd.c_str());
                } else if (tok.compare(0, 16, "gangdomainlevel=") == 0) {
                    pod.Requests[GPUGangDomainLevel] = atoll(tok.c_str() + 16);
                } else if (tok.compare(0, 9, "priority=") == 0) {
                    pod.Requests[GPUPriorityLevel] = atoll(tok.c_str() + 9);
                } else if (cur && tok.compare(0, 4, "req=") == 0) {
                    cur->Requests[gpuplugintypes::ResourceGPU] = atoll(tok.c_str() + 4);
                } else if (cur && tok.compare(0, 5, "kube=") == 0) {
                    cur->KubeRequests[gpuplugintypes::ResourceGPU] = atoll(tok.c_str() + 5);
                } else if (cur && tok.compare(0, 4, "dev:") == 0 && splitKV(tok.substr(4), &k, &v)) {
                    cur->DevRequests[k] = v;
                }
            }
        } else if (cmd == "fits" || cmd == "allocate") {
            std::string node, podName;
            in >> node >> podName;
            if (!g_nodes.count(node) || !g_pods.count(podName)) { printf("  unknown node or pod\n"); continue; }
            types::PodInfo &pod = g_pods[podName];
            if (cmd == "fits") {
                double score = -1.0;
                std::vector<kubedevice::devicescheduler::PredicateFailureReason> reasons;
                const bool fits = sched.PodFitsDevice(&g_nodes[node], &pod, false, &reasons, &score);
                printf("  fits=%d reasons=%zu score=%.17g\n", fits ? 1 : 0, reasons.size(), score);
            } else {
                printf("  err=%s\n", sched.PodAllocate(&g_nodes[node], &pod).c_str());
            }
            dumpPod(pod);
        } else if (cmd == "take" || cmd == "return") {
            std::string podName;
            in >> podName;
            if (!g_pods.count(podName)) { printf("  unknown pod\n"); continue; }
            const std::string err = cmd == "take" ? sched.TakePodResources(nullptr, &g_pods[podName])
                                                  : sched.ReturnPodResources(nullptr, &g_pods[podName]);
            printf("  err=%s\n", err.c_str());
        } else if (cmd == "using") {
            printf("  UsingGroupScheduler=%d name=%s\n", sched.UsingGroupScheduler() ? 1 : 0, sched.GetName().c_str());
        } else if (cmd == "scorebatch" || cmd == "placebatch" || cmd == "proposebatch") {
            std::vector<const types::PodInfo *> pods;
            std::string podName;
            while (in >> podName)
                if (g_pods.count(podName)) pods.push_back(&g_pods[podName]);
            std::vector<Placement> out;
            const std::string err = cmd == "placebatch"     ? sched.PlaceBatch(pods, &out)
                                    : cmd == "proposebatch" ? sched.ProposeBatch(pods, &out)
                                                            : sched.ScoreBatch(pods, &out);
            printf("  err=%s\n", err.c_str());
            for (size_t i = 0; i < out.size(); i++)
                printf("  %s fits=%d cost=%u node=%s mask=0x%02x\n", pods[i]->Name.c_str(), out[i].fits ? 1 : 0, out[i].cost,
                       out[i].nodeName.c_str(), out[i].gpuMask);
        } else if (cmd == "preemptbatch" || cmd == "preemptplan" || cmd == "preemptgangplan" ||
                   cmd == "preemptdomainplan") {
            std::vector<const types::PodInfo *> pods;
            std::string podName;
            while (in >> podName)
                if (g_pods.count(podName)) pods.push_back(&g_pods[podName]);
            std::vector<Placement> out;
            std::vector<std::vector<std::string>> victims;
            const std::string err = cmd == "preemptplan"       ? sched.PlanPreemption(pods, &out, &victims)
                                    : cmd == "preemptgangplan" ? sched.PlanGangPreemption(pods, &out, &victims)
                                    : cmd == "preemptdomainplan" ? sched.PlanGangDomainPreemption(pods, &out, &victims)
                                                               : sched.PreemptBatch(pods, &out, &victims);
            printf("  err=%s\n", err.c_str());
            for (size_t i = 0; i < out.size(); i++) {
                std::string names;
                for (const std::string &v : victims[i]) names += (names.empty() ? "" : ",") + v;
                printf("  %s fits=%d cost=%u node=%s mask=0x%02x victims=%s\n", pods[i]->Name.c_str(), out[i].fits ? 1 : 0,
                       out[i].cost, out[i].nodeName.c_str(), out[i].gpuMask, names.c_str());
            }
        } else if (cmd == "cache") {
            // sorted by (tree text) so the transcript does not depend on insertion order
            std::vector<std::string> rows;
            for (const auto &e : sched.cache().entries()) {
                std::string row = gpuplugintypes::FormatTreeNode(e->tree.get());
                char buf[64];
                snprintf(buf, sizeof buf, "score=%.17g nodes=", e->TreeScore);
                row += buf;
                for (const auto &n : e->ListOfNodes) row += n.first + ",";
                rows.push_back(row);
            }
            std::sort(rows.begin(), rows.end());
            for (const auto &r : rows) printf("%s\n", r.c_str());
        } else if (cmd == "best") {
            int k = 0;
            in >> k;
            const SortedTreeNode *t = sched.cache().findBestTreeInCache(k);
            printf("%s", t ? gpuplugintypes::FormatTreeNode(t).c_str() : "  none\n");
        } else {
            printf("  unknown command\n");
        }
    }
    return 0;
}
