// host_pods_test.cc -- the Provider's pending-pod tick selects by slot (rpk_select_slots) from the device pod table, and
// seeds only the rows whose columns changed since the last tick.  The columns are still derived from the annotations on
// every tick, so a changed pod annotation, a changed owner-Job annotation and a reused slot all reach the selection, and
// every pod gets the gpuTypeIds that PrepareColumnsBatch + rpk_select give it.  Needs a GPU (the Provider refuses to
// start without one).
#include <cstdio>
#include <map>
#include <mutex>
#include <random>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

struct RecordingRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;
    bool fail_deploy = false, fail_fetch = false;
    int deploys = 0;
    std::map<std::string, std::vector<std::string>> ids_of;  // pod name -> gpuTypeIds of its last deploy attempt
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        if (fail_fetch) { *err = "graphql down"; return false; }
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const std::vector<std::string>& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        ids_of[pod.name] = ids;
        if (fail_deploy || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
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

static PodPtr MakePod(const std::string& name, Annotations ann = {}, std::shared_ptr<Annotations> job = nullptr) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending"; p->annotations = std::move(ann); p->owner_job = std::move(job);
    return p;
}

static void TestSeedsOnlyWhatChanged() {
    auto api = std::make_shared<RecordingRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 256);
    api->fail_fetch = true;  // CreatePod's deploy stops before the selection: nothing is seeded yet
    for (int i = 0; i < 40; ++i) prov.CreatePod(MakePod("pend" + std::to_string(i), {{GpuMemoryAnnotation, i % 2 ? "24" : "48"}}));
    api->fail_fetch = false;
    CHECK_EQ(prov.PodSeeds(), 0u);
    api->fail_deploy = true;  // the pods stay pending
    uint64_t sel = prov.SelectCalls(), seeds = prov.PodSeeds();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.SelectCalls(), sel + 1);  // ONE rpk_select_slots for the batch
    CHECK_EQ(prov.PodSeeds(), seeds + 40);  // every row differs from the no-annotation default
    CHECK_EQ(api->ids_of.size(), 40u);
    for (auto& kv : api->ids_of) CHECK_EQ(kv.second, std::stoi(kv.first.substr(4)) % 2 ? kIds24 : kIds48);
    sel = prov.SelectCalls(); seeds = prov.PodSeeds();
    prov.ProcessPendingPods();  // nothing changed: no seed, still one select
    CHECK_EQ(prov.SelectCalls(), sel + 1);
    CHECK_EQ(prov.PodSeeds(), seeds);

    // UpdatePod changing the memory annotation re-seeds exactly that slot, and the deploy follows the new value
    prov.UpdatePod(MakePod("pend7", {{GpuMemoryAnnotation, "48"}}));
    seeds = prov.PodSeeds();
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PodSeeds(), seeds + 1);
    CHECK_EQ(api->ids_of["pend7"], kIds48);
    CHECK_EQ(api->ids_of["pend9"], kIds24);
    // ... and back to 24 GB once deploys work again: the pods deploy with the ids of their current columns
    prov.UpdatePod(MakePod("pend7", {{GpuMemoryAnnotation, "24"}}));
    api->fail_deploy = false;
    api->ids_of.clear();
    seeds = prov.PodSeeds();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PodSeeds(), seeds + 1);
    CHECK_EQ(api->ids_of["pend7"], kIds24);
    CHECK_EQ(api->ids_of.size(), 40u);
    CHECK(prov.GetPod("default", "pend7").first->annotations.count(PodIDAnnotation) == 1);
}

static void TestOwnerJobAndSlotReuse() {
    auto api = std::make_shared<RecordingRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 64);
    api->fail_deploy = true;
    auto job = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "24"}});
    prov.CreatePod(MakePod("jobpod", {}, job));  // the owner Job's annotation is the pod's column (runpod_client.go:1102-1112)
    CHECK_EQ(api->ids_of["jobpod"], kIds24);
    (*job)[GpuMemoryAnnotation] = "48";           // the Job changes; the pod object does not
    uint64_t seeds = prov.PodSeeds();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.PodSeeds(), seeds + 1);
    CHECK_EQ(api->ids_of["jobpod"], kIds48);

    // a slot freed by DeletePod and handed to the next pod holds the new pod's columns, not the old one's
    prov.CreatePod(MakePod("old", {{GpuMemoryAnnotation, "48"}}));
    CHECK_EQ(api->ids_of["old"], kIds48);
    prov.DeletePod(prov.GetPod("default", "old").first);
    seeds = prov.PodSeeds();
    prov.CreatePod(MakePod("new"));  // no annotations: 16 GB, SECURE
    CHECK_EQ(prov.PodSeeds(), seeds + 1);
    CHECK_EQ(api->ids_of["new"], kIds16);
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(api->ids_of["new"], kIds16);
    CHECK_EQ(api->ids_of["jobpod"], kIds48);
}

// A random population: every pod's gpuTypeIds from the Provider's slot select equals PrepareColumnsBatch + rpk_select over
// the same pods, through creation, updates, deletions and slot reuse.
static void TestRandomPopulation() {
    std::mt19937 rng(7);
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
    std::vector<std::shared_ptr<Annotations>> jobs;
    for (int j = 0; j < 8; ++j)
        jobs.push_back(std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, mems[rng() % 9]}, {CloudTypeAnnotation, clouds[rng() % 4]}}));
    auto random_pod = [&](const std::string& name) {
        Annotations a;
        auto put = [&](const char* key, const char* v) { if (*v) a[key] = v; };
        put(GpuMemoryAnnotation, mems[rng() % 9]); put(CloudTypeAnnotation, clouds[rng() % 4]); put(MaxPriceAnnotation, prices[rng() % 6]);
        if (rng() % 3 == 0) a[VcpuAnnotation] = std::to_string(4 * (rng() % 6));
        if (rng() % 3 == 0) a[RamAnnotation] = std::to_string(16 * (rng() % 6));
        return MakePod(name, std::move(a), rng() % 4 == 0 ? jobs[rng() % jobs.size()] : nullptr);
    };
    const int kPods = 2000;
    Provider prov(api, 1, 4096);
    api->fail_deploy = true;  // everybody stays pending; DeployPod still records the ids each pod was offered
    api->fail_fetch = true;
    std::vector<std::string> names;
    for (int i = 0; i < kPods; ++i) { names.push_back("r" + std::to_string(i)); prov.CreatePod(random_pod(names.back())); }
    api->fail_fetch = false;
    int next = kPods;
    for (int round = 0; round < 3; ++round) {
        api->ids_of.clear();
        prov.ProcessPendingPods();
        std::vector<PodPtr> pods;
        for (const auto& n : names) pods.push_back(prov.GetPod("default", n).first);
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
            auto it = api->ids_of.find(names[i]);
            if (it == api->ids_of.end() || it->second != want) ++bad;
        }
        CHECK_EQ(bad, 0);
        CHECK_EQ(api->ids_of.size(), (size_t)P);
        // churn: update 300 pods, change two Jobs, delete 200 pods and create 200 new ones in the freed slots
        for (int k = 0; k < 300; ++k) prov.UpdatePod(random_pod(names[rng() % names.size()]));
        (*jobs[0])[GpuMemoryAnnotation] = mems[rng() % 9]; (*jobs[1])[CloudTypeAnnotation] = clouds[rng() % 4];
        for (int k = 0; k < 200; ++k) {
            const size_t victim = rng() % names.size();
            prov.DeletePod(prov.GetPod("default", names[victim]).first);
            names[victim] = "r" + std::to_string(next++);
            prov.CreatePod(random_pod(names[victim]));
        }
    }
    std::printf("random population: %d pods, %llu rows seeded over 3 ticks + churn\n", kPods, (unsigned long long)prov.PodSeeds());
}

int main() {
    TestSeedsOnlyWhatChanged();
    TestOwnerJobAndSlotReuse();
    TestRandomPopulation();
    std::printf("%s: %d checks, %d failed (gpu)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
