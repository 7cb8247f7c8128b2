// host_pending_test.cc -- the Provider's pending-pod tick keeps the set of pending slots on the device: it uploads only
// the pending flags that changed (rpk_pods_mark_pending), sends no slot list, and selects with rpk_select_pending.  A
// deployed, deleted or failed pod leaves the set, a reused slot is marked again, a pod created or deployed by another
// thread while a tick runs is neither lost nor deployed twice, and every pending pod of a random population with churn
// gets the gpuTypeIds that PrepareColumnsBatch + rpk_select give it.  Needs a GPU (the Provider refuses to start
// without one).
#include <cstdio>
#include <functional>
#include <map>
#include <mutex>
#include <random>
#include <set>
#include <thread>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

struct RecordingRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;
    bool fail_fetch = false;
    std::function<bool(const std::string&)> refuses = [](const std::string&) { return false; };  // pods whose deploy fails
    std::function<void()> on_fetch;                       // called (unlocked) from FetchGPUTypes
    std::function<void(const std::string&)> on_deploy;    // called (unlocked) from DeployPod, before it answers
    int deploys = 0;
    std::map<std::string, std::vector<std::string>> ids_of;  // pod name -> gpuTypeIds of its last deploy attempt
    std::map<std::string, int> attempts, deployed;           // pod name -> DeployPod calls, successful ones
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string* err) override {
        if (on_fetch) on_fetch();
        std::lock_guard<std::mutex> g(mu);
        if (fail_fetch) { *err = "graphql down"; return false; }
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const std::vector<std::string>& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        if (on_deploy) on_deploy(pod.name);
        std::lock_guard<std::mutex> g(mu);
        ids_of[pod.name] = ids; ++attempts[pod.name];
        if (refuses(pod.name) || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25; ++deployed[pod.name];
        return true;
    }
    bool GetDetailedPodStatus(const std::string&, DetailedStatus*, std::string* err) override { *err = "http 500"; return false; }
    bool TerminatePod(const std::string&, std::string*) override { return true; }
};

static std::vector<GPUType> KatTable() {  // tests/golden/select_kat.json
    return {{"A4000", "", 16, true, .32, true, .17}, {"A5000", "", 24, true, .36, true, .22}, {"RTX3090", "", 24, false, 0, true, .22},
            {"A40", "", 48, true, .40, false, 0},    {"RTX4090", "", 24, true, .69, true, .34}, {"L4", "", 24, true, .43, false, 0},
            {"A100", "", 80, true, 1.64, true, 1.19}, {"T4free", "", 16, true, 0, true, 0},     {"A4500", "", 20, true, .34, true, .19},
            {"edge", "", 32, true, .5, true, .5}};
}
using Ids = std::vector<std::string>;
static const Ids kIds16 = {"A4000", "A4500", "A5000", "A40", "L4"}, kIds24 = {"A5000", "A40", "L4"}, kIds48 = {"A40"};
static const auto kAll = [](const std::string&) { return true; };
static const auto kNone = [](const std::string&) { return false; };

static PodPtr MakePod(const std::string& name, Annotations ann = {}, std::shared_ptr<Annotations> job = nullptr) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending"; p->annotations = std::move(ann); p->owner_job = std::move(job);
    return p;
}

static void TestMarksOnlyWhatChanged() {
    auto api = std::make_shared<RecordingRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 256);
    api->refuses = kAll;  // the pods stay pending
    for (int i = 0; i < 40; ++i) prov.CreatePod(MakePod("pend" + std::to_string(i), {{GpuMemoryAnnotation, i % 2 ? "24" : "48"}}));
    CHECK_EQ(prov.PendingMarks(), 0u);  // CreatePod selects its own pod by slot; flags go up with the tick
    uint64_t sel = prov.SelectCalls();
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 40u);
    CHECK_EQ(prov.SelectCalls(), sel + 1);  // ONE rpk_select_pending for the batch
    CHECK_EQ(api->ids_of.size(), 40u);
    for (auto& kv : api->ids_of) CHECK_EQ(kv.second, std::stoi(kv.first.substr(4)) % 2 ? kIds24 : kIds48);
    prov.ProcessPendingPods();  // nothing entered or left the set
    CHECK_EQ(prov.PendingMarks(), 40u);
    CHECK_EQ(prov.SelectCalls(), sel + 2);

    // the odd pods deploy: they leave the set, and the next tick offers the even ones only
    api->refuses = [](const std::string& n) { return n.rfind("pend", 0) != 0 || std::stoi(n.substr(4)) % 2 == 0; };
    prov.ProcessPendingPods();
    CHECK_EQ(api->deploys, 20);
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 60u);  // 20 flags cleared
    CHECK_EQ(api->ids_of.size(), 20u);
    CHECK_EQ(api->ids_of.count("pend1"), 0u);
    CHECK_EQ(api->ids_of["pend0"], kIds48);

    // a deleted pod leaves the set
    prov.DeletePod(prov.GetPod("default", "pend0").first);
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 61u);
    CHECK_EQ(api->ids_of.size(), 19u);
    // its slot goes to the next pod, which is marked again
    prov.CreatePod(MakePod("heir"));
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 62u);
    CHECK_EQ(api->ids_of["heir"], kIds16);
    CHECK_EQ(api->ids_of.size(), 20u);
    // ... and a slot reused between two ticks keeps its flag: nothing to upload, the new pod's columns are selected
    prov.DeletePod(prov.GetPod("default", "heir").first);
    prov.CreatePod(MakePod("heir2", {{GpuMemoryAnnotation, "24"}}));
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 62u);
    CHECK_EQ(api->ids_of["heir2"], kIds24);
    CHECK_EQ(api->ids_of.count("heir"), 0u);

    // an UpdatePod that carries a RunPod id, or another phase, takes the pod out; one that drops the id brings it back
    prov.UpdatePod(MakePod("pend2", {{GpuMemoryAnnotation, "48"}, {PodIDAnnotation, "rp-elsewhere"}}));
    auto running = MakePod("pend4", {{GpuMemoryAnnotation, "48"}});
    running->status.phase = "Running";
    prov.UpdatePod(running);
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 64u);
    CHECK_EQ(api->ids_of.count("pend2") + api->ids_of.count("pend4"), 0u);
    prov.UpdatePod(MakePod("pend2", {{GpuMemoryAnnotation, "48"}}));
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PendingMarks(), 65u);
    CHECK_EQ(api->ids_of["pend2"], kIds48);

    // after 15 minutes the remaining pods are failed: tried once more, then out of the set and not selected again
    prov.SetClock(16 * 60);
    prov.ProcessPendingPods();
    CHECK_EQ(prov.GetPod("default", "pend6").first->status.phase, std::string("Failed"));
    sel = prov.SelectCalls();
    const uint64_t marks = prov.PendingMarks();
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK(prov.PendingMarks() > marks);
    CHECK_EQ(api->ids_of.size(), 0u);
    CHECK_EQ(prov.SelectCalls(), sel);  // nothing pending: no select
}

// Another thread creates a pod while a tick is between its flag upload and its select; and a pod of the batch gets its
// RunPod id from elsewhere before the tick reaches it.
static void TestPodsThatChangeDuringATick() {
    auto api = std::make_shared<RecordingRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 64);
    api->refuses = kAll;
    for (int i = 0; i < 6; ++i) prov.CreatePod(MakePod("p" + std::to_string(i), {{GpuMemoryAnnotation, "24"}}));
    api->refuses = kNone;
    std::thread creator;
    bool spawned = false;
    api->on_fetch = [&] {  // the tick holds the engine here, its flags already uploaded: the creator waits for the select
        if (spawned) return;
        spawned = true;
        creator = std::thread([&] { prov.CreatePod(MakePod("late", {{GpuMemoryAnnotation, "48"}})); });
    };
    api->on_deploy = [&](const std::string& name) {  // while the tick deploys its first pod, p5 is deployed elsewhere
        if (name == "p0") prov.UpdatePod(MakePod("p5", {{GpuMemoryAnnotation, "24"}, {PodIDAnnotation, "rp-elsewhere"}}));
    };
    prov.ProcessPendingPods();
    creator.join();
    api->on_fetch = nullptr; api->on_deploy = nullptr;
    CHECK_EQ(api->deployed["late"], 1);  // by its own CreatePod
    CHECK_EQ(api->ids_of["late"], kIds48);
    CHECK_EQ(api->attempts["p5"], 1);  // only the attempt of its CreatePod: the tick skipped it
    for (int i = 0; i < 5; ++i) CHECK_EQ(api->deployed["p" + std::to_string(i)], 1);
    const int deploys = api->deploys;
    prov.ProcessPendingPods();  // everybody has an id: the flags are cleared, nobody is deployed twice
    prov.ProcessPendingPods();
    CHECK_EQ(api->deploys, deploys);
    CHECK_EQ(api->attempts["late"], 1);
}

// A random population over several ticks: some pods deploy and leave, pods are updated, deleted and created in reused
// slots; every tick, every pending pod is offered exactly the gpuTypeIds of PrepareColumnsBatch + rpk_select, and nobody
// else is offered anything.
static void TestRandomPopulation() {
    std::mt19937 rng(11);
    auto api = std::make_shared<RecordingRunPod>();
    for (int g = 0; g < 300; ++g) {
        GPUType t;
        t.ID = "gpu" + std::to_string(g);
        t.MemoryInGb = 8 * (1 + (int)(rng() % 12)); t.VCPU = 4 * (int)(rng() % 9); t.RAMGb = 16 * (int)(rng() % 9);
        t.SecureCloud = rng() % 4 != 0; t.CommunityCloud = rng() % 3 != 0;
        t.SecurePrice = (double)(rng() % 200) / 100.0; t.CommunityPrice = (double)(rng() % 150) / 100.0;
        api->types.push_back(t);
    }
    const char* mems[] = {"", "8", "16", "24", "40", "48", "80", "96", "abc"};
    const char* clouds[] = {"", "SECURE", "COMMUNITY", "STANDARD"};
    const char* prices[] = {"", "0.3", "0.5", "0.9", "1.5", "cheap"};
    auto random_pod = [&](const std::string& name) {
        Annotations a;
        auto put = [&](const char* key, const char* v) { if (*v) a[key] = v; };
        put(GpuMemoryAnnotation, mems[rng() % 9]); put(CloudTypeAnnotation, clouds[rng() % 4]); put(MaxPriceAnnotation, prices[rng() % 6]);
        if (rng() % 3 == 0) a[VcpuAnnotation] = std::to_string(4 * (rng() % 6));
        if (rng() % 3 == 0) a[RamAnnotation] = std::to_string(16 * (rng() % 6));
        return MakePod(name, std::move(a));
    };
    const int kPods = 6000;  // above the select's latency path
    Provider prov(api, 1, 8192);
    int round = 0;
    // a pod's deploy works in the round its number picks (a fifth of them per round), never for the rest
    api->refuses = [&](const std::string& n) { return std::stoi(n.substr(1)) % 5 != round; };
    api->fail_fetch = true;
    std::set<std::string> names;
    for (int i = 0; i < kPods; ++i) { names.insert("r" + std::to_string(i)); prov.CreatePod(random_pod("r" + std::to_string(i))); }
    api->fail_fetch = false;
    int next = kPods;
    for (; round < 4; ++round) {
        std::vector<std::string> pending;  // by the predicate, before the tick
        std::vector<PodPtr> pods;
        for (const auto& n : names) {
            PodPtr p = prov.GetPod("default", n).first;
            if (p->status.phase == "Pending" && !p->annotations.count(PodIDAnnotation)) { pending.push_back(n); pods.push_back(p); }
        }
        api->ids_of.clear();
        prov.ProcessPendingPods();
        PodColumnsSoA cols;
        PrepareColumnsBatch(pods, &cols);
        const uint32_t P = (uint32_t)pods.size();
        std::vector<int32_t> best(P), top5((size_t)P * RPK_TOPK);
        CHECK_EQ(rpk_select(prov.Ctx(), P, cols.req_mem_gb.data(), cols.req_vcpu.data(), cols.req_ram_gb.data(), cols.max_price.data(),
                            cols.cloud.data(), best.data(), top5.data()), RPK_OK);
        int bad = 0;
        for (uint32_t i = 0; i < P; ++i) {
            Ids want;
            for (int k = 0; k < RPK_TOPK; ++k) { const int32_t g = top5[(size_t)i * RPK_TOPK + k]; if (g >= 0) want.push_back(api->types[(size_t)g].ID); }
            auto it = api->ids_of.find(pending[i]);
            if (it == api->ids_of.end() || it->second != want) ++bad;
        }
        CHECK_EQ(bad, 0);
        CHECK_EQ(api->ids_of.size(), (size_t)P);  // nobody outside the set was offered anything
        CHECK(P > 1000);
        // churn: update 300 pods (some of them deployed ones, which stay out), delete 200 and create 200 in the freed slots
        for (int k = 0; k < 300; ++k) {
            auto it = names.begin();
            std::advance(it, rng() % names.size());
            PodPtr cur = prov.GetPod("default", *it).first, up = random_pod(*it);
            if (cur->annotations.count(PodIDAnnotation)) up->annotations[PodIDAnnotation] = cur->annotations.at(PodIDAnnotation);
            prov.UpdatePod(up);
        }
        api->fail_fetch = true;  // the new pods wait for the tick
        for (int k = 0; k < 200; ++k) {
            auto it = names.begin();
            std::advance(it, rng() % names.size());
            prov.DeletePod(prov.GetPod("default", *it).first);
            names.erase(it);
            const std::string fresh = "r" + std::to_string(next++);
            names.insert(fresh);
            prov.CreatePod(random_pod(fresh));
        }
        api->fail_fetch = false;
    }
    std::printf("random population: %d pods, %llu flags marked, %llu rows seeded, %d deployed over 4 ticks + churn\n", kPods,
                (unsigned long long)prov.PendingMarks(), (unsigned long long)prov.PodSeeds(), api->deploys);
}

int main() {
    TestMarksOnlyWhatChanged();
    TestPodsThatChangeDuringATick();
    TestRandomPopulation();
    std::printf("%s: %d checks, %d failed (gpu)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
