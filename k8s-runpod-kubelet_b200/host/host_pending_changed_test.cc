// host_pending_changed_test.cc -- the Provider's pending tick with rpk_select_pending_changed: it keeps a per-slot mirror
// of the top-5 offer indices the call reports, and deploys every pending pod from it.  Over ticks with churn and offer
// refreshes every DeployPod gets the gpuTypeIds a reference select of the same pods gives; a steady tick recomputes no
// row; a refresh that changes one price changes only the affected pods' lists; a slot reused by another pod with
// identical columns deploys with the right ids.  Needs a GPU (the Provider refuses to start without one).
#include <cstdio>
#include <functional>
#include <map>
#include <mutex>
#include <random>
#include <set>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

using Ids = std::vector<std::string>;

struct RecordingRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;
    std::function<bool(const std::string&)> refuses = [](const std::string&) { return true; };  // pods whose deploy fails
    int deploys = 0;
    std::map<std::string, Ids> ids_of;  // pod name -> gpuTypeIds of its last deploy attempt
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string*) override {
        std::lock_guard<std::mutex> g(mu);
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const Ids& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        ids_of[pod.name] = ids;
        if (refuses(pod.name) || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
        return true;
    }
    bool GetDetailedPodStatus(const std::string&, DetailedStatus*, std::string* err) override { *err = "http 500"; return false; }
    bool TerminatePod(const std::string&, std::string*) override { return true; }
};

static PodPtr MakePod(const std::string& name, Annotations ann = {}) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending"; p->annotations = std::move(ann);
    return p;
}

struct Population {
    std::mt19937 rng{23};
    std::shared_ptr<RecordingRunPod> api = std::make_shared<RecordingRunPod>();
    std::set<std::string> names;
    Population() {
        for (int g = 0; g < 300; ++g) {
            GPUType t;
            t.ID = "gpu" + std::to_string(g);
            t.MemoryInGb = 8 * (1 + (int)(rng() % 12)); t.VCPU = 4 * (int)(rng() % 9); t.RAMGb = 16 * (int)(rng() % 9);
            t.SecureCloud = rng() % 4 != 0; t.CommunityCloud = rng() % 3 != 0;
            t.SecurePrice = (double)(rng() % 200) / 100.0; t.CommunityPrice = (double)(rng() % 150) / 100.0;
            api->types.push_back(t);
        }
    }
    PodPtr Random(const std::string& name) {
        static const char* mems[] = {"", "8", "16", "24", "40", "48", "80", "96"};
        static const char* clouds[] = {"", "SECURE", "COMMUNITY"};
        static const char* prices[] = {"", "0.3", "0.5", "0.9", "1.5"};
        Annotations a;
        auto put = [&](const char* key, const char* v) { if (*v) a[key] = v; };
        put(GpuMemoryAnnotation, mems[rng() % 8]); put(CloudTypeAnnotation, clouds[rng() % 3]); put(MaxPriceAnnotation, prices[rng() % 5]);
        if (rng() % 3 == 0) a[VcpuAnnotation] = std::to_string(4 * (rng() % 6));
        return MakePod(name, std::move(a));
    }
    // the pending pods before a tick, and what a reference select of their columns offers each
    std::map<std::string, Ids> Reference(Provider& prov) {
        std::vector<std::string> pending;
        std::vector<PodPtr> pods;
        for (const auto& n : names) {
            PodPtr p = prov.GetPod("default", n).first;
            if (p->status.phase == "Pending" && !p->annotations.count(PodIDAnnotation)) { pending.push_back(n); pods.push_back(p); }
        }
        PodColumnsSoA cols;
        PrepareColumnsBatch(pods, &cols);
        const uint32_t P = (uint32_t)pods.size();
        std::vector<int32_t> best(P), top5((size_t)P * RPK_TOPK);
        std::vector<GPUType> types;
        { std::lock_guard<std::mutex> g(api->mu); types = api->types; }
        std::map<std::string, Ids> want;
        if (P == 0) return want;
        // the offers as the tick will see them: the Provider refreshes its table from the fake first
        std::vector<int32_t> mem, vcpu, ram;
        std::vector<double> sp, cp;
        std::vector<uint8_t> fl;
        for (const auto& t : types) {
            mem.push_back(t.MemoryInGb); vcpu.push_back(t.VCPU); ram.push_back(t.RAMGb); sp.push_back(t.SecurePrice); cp.push_back(t.CommunityPrice);
            fl.push_back((uint8_t)((t.SecureCloud ? RPK_FLAG_SECURE_CLOUD : 0u) | (t.CommunityCloud ? RPK_FLAG_COMMUNITY_CLOUD : 0u)));
        }
        rpk_ctx* ref = nullptr;
        CHECK_EQ(rpk_create(1, nullptr, &ref), RPK_OK);
        CHECK_EQ(rpk_offers_upload(ref, (uint32_t)types.size(), mem.data(), vcpu.data(), ram.data(), sp.data(), cp.data(), fl.data()), RPK_OK);
        std::vector<uint32_t> slots(P);
        for (uint32_t i = 0; i < P; ++i) slots[i] = i;
        CHECK_EQ(rpk_pods_reset(ref, P), RPK_OK);
        CHECK_EQ(rpk_pods_seed_slots(ref, P, slots.data(), cols.req_mem_gb.data(), cols.req_vcpu.data(), cols.req_ram_gb.data(),
                                     cols.max_price.data(), cols.cloud.data()), RPK_OK);
        CHECK_EQ(rpk_select_slots(ref, P, slots.data(), best.data(), top5.data()), RPK_OK);
        rpk_destroy(ref);
        for (uint32_t i = 0; i < P; ++i) {
            Ids& w = want[pending[i]];
            for (int k = 0; k < RPK_TOPK; ++k) { const int32_t g = top5[(size_t)i * RPK_TOPK + k]; if (g >= 0) w.push_back(types[(size_t)g].ID); }
        }
        return want;
    }
};

// every tick's deploys equal the reference; steady ticks recompute nothing; a one-price refresh reports only what changed
static void TestTicksMatchTheReference() {
    Population pop;
    auto& api = pop.api;
    const int kPods = 5000;  // above the select's latency path
    Provider prov(api, 1, 8192);
    for (int i = 0; i < kPods; ++i) { pop.names.insert("r" + std::to_string(i)); prov.CreatePod(pop.Random("r" + std::to_string(i))); }
    int next = kPods;
    for (int round = 0; round < 6; ++round) {
        const std::map<std::string, Ids> want = pop.Reference(prov);
        api->ids_of.clear();
        const uint64_t sel = prov.SelectCalls(), rows = prov.ReselectedRows(), lists = prov.ChangedLists();
        prov.ProcessPendingPods();
        CHECK(api->ids_of == want);
        CHECK_EQ(prov.SelectCalls(), sel + 1);
        CHECK(prov.ChangedLists() - lists <= prov.ReselectedRows() - rows);
        // a steady tick: the same pods, nothing recomputed, the same lists
        const uint64_t rows2 = prov.ReselectedRows();
        api->ids_of.clear();
        prov.ProcessPendingPods();
        CHECK_EQ(prov.ReselectedRows(), rows2);
        CHECK(api->ids_of == want);
        if (round == 2) {  // one price changes: only the pods whose list changes get a new list back
            int g = 0;
            for (const auto& kv : want) if (!kv.second.empty()) { g = std::stoi(kv.second[0].substr(3)); break; }
            { std::lock_guard<std::mutex> lk(api->mu); api->types[(size_t)g].SecurePrice *= 0.5; api->types[(size_t)g].CommunityPrice *= 0.5; }
            const std::map<std::string, Ids> want2 = pop.Reference(prov);
            size_t differ = 0;
            for (const auto& kv : want2) differ += want.at(kv.first) != kv.second;
            const uint64_t l0 = prov.ChangedLists(), r0 = prov.ReselectedRows();
            api->ids_of.clear();
            prov.ProcessPendingPods();
            CHECK(api->ids_of == want2);
            CHECK_EQ(prov.ChangedLists() - l0, (uint64_t)differ);
            CHECK_EQ(prov.ReselectedRows() - r0, (uint64_t)want2.size());  // a new table: every pending row
            CHECK(differ > 0 && differ < want2.size());
        }
        // churn: a tenth deploys, 200 updates, 150 deletes and creates
        api->refuses = [round](const std::string& n) { return std::stoi(n.substr(1)) % 10 != round; };
        prov.ProcessPendingPods();
        api->refuses = [](const std::string&) { return true; };
        for (int k = 0; k < 200; ++k) {
            auto it = pop.names.begin();
            std::advance(it, pop.rng() % pop.names.size());
            PodPtr cur = prov.GetPod("default", *it).first, up = pop.Random(*it);
            if (cur->annotations.count(PodIDAnnotation)) up->annotations[PodIDAnnotation] = cur->annotations.at(PodIDAnnotation);
            prov.UpdatePod(up);
        }
        for (int k = 0; k < 150; ++k) {
            auto it = pop.names.begin();
            std::advance(it, pop.rng() % pop.names.size());
            prov.DeletePod(prov.GetPod("default", *it).first);
            pop.names.erase(it);
            const std::string fresh = "r" + std::to_string(next++);
            pop.names.insert(fresh);
            prov.CreatePod(pop.Random(fresh));
        }
    }
    std::printf("ticks: %llu rows reselected, %llu lists changed, %d deployed\n", (unsigned long long)prov.ReselectedRows(),
                (unsigned long long)prov.ChangedLists(), api->deploys);
}

// a slot freed by one pod and taken by another with identical columns: nothing is recomputed, and the new pod deploys
// with the list its columns give
static void TestReusedSlotWithIdenticalColumns() {
    Population pop;
    auto& api = pop.api;
    Provider prov(api, 1, 64);
    for (int i = 0; i < 20; ++i) { pop.names.insert("p" + std::to_string(i)); prov.CreatePod(MakePod("p" + std::to_string(i), {{GpuMemoryAnnotation, i % 2 ? "24" : "48"}})); }
    prov.ProcessPendingPods();
    prov.DeletePod(prov.GetPod("default", "p3").first);
    pop.names.erase("p3");
    pop.names.insert("heir");
    prov.CreatePod(MakePod("heir", {{GpuMemoryAnnotation, "24"}}));  // p3's columns
    const std::map<std::string, Ids> want = pop.Reference(prov);
    const uint64_t rows = prov.ReselectedRows();
    api->ids_of.clear();
    prov.ProcessPendingPods();
    CHECK(api->ids_of == want);
    CHECK(!api->ids_of["heir"].empty());
    CHECK_EQ(prov.ReselectedRows(), rows);
}

int main() {
    TestTicksMatchTheReference();
    TestReusedSlotWithIdenticalColumns();
    std::printf("%s: %d checks, %d failed (gpu)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
