// host_grow_test.cc -- a Provider whose pods outgrow its initial capacity doubles it in place instead of refusing the
// pod.  A Provider starting at 16 slots takes 5 000 pods over many pending ticks and sweeps, with deploy failures and
// status churn: nothing throws, every pending pod deploys with the gpuTypeIds a reference select of its columns gives,
// a steady tick recomputes nothing, and the deploys, the rows reselected and the notifications (every status
// transition, in order) are those of a Provider built with 8 192 slots, which never grows.  Then one thread creates and deletes pods while
// another sweeps, across several growths.  Needs a GPU (the Provider refuses to start without one).
#include <atomic>
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

using Ids = std::vector<std::string>;

struct FakeRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;
    std::function<bool(const std::string&)> refuses = [](const std::string&) { return true; };  // pods whose deploy fails
    int deploys = 0;
    std::map<std::string, Ids> ids_of;           // pod name -> gpuTypeIds of its last deploy attempt
    std::map<std::string, std::string> status;   // RunPod id -> DesiredStatus
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string*) override {
        std::lock_guard<std::mutex> g(mu);
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const Ids& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        ids_of[pod.name] = ids;
        if (refuses(pod.name) || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
        status[*id] = "CREATED";
        return true;
    }
    bool GetDetailedPodStatus(const std::string& id, DetailedStatus* out, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        auto it = status.find(id);
        if (it == status.end()) { *err = "http 500"; return false; }
        out->DesiredStatus = it->second;
        return true;
    }
    bool TerminatePod(const std::string&, std::string*) override { return true; }
    void SetStatus(const std::string& id, const std::string& s) { std::lock_guard<std::mutex> g(mu); status[id] = s; }
};

static PodPtr MakePod(const std::string& name, Annotations ann = {}) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending"; p->annotations = std::move(ann);
    return p;
}

// One Provider and everything it is driven with.  Two Worlds with the same seed see the same calls.
struct World {
    std::mt19937 rng{31};
    std::shared_ptr<FakeRunPod> api = std::make_shared<FakeRunPod>();
    std::set<std::string> names;
    std::vector<std::string> notes;  // "name:phase" per notification, in order
    Provider prov;
    explicit World(uint32_t slots) : prov(api, 1, slots) {
        for (int g = 0; g < 300; ++g) {
            GPUType t;
            t.ID = "gpu" + std::to_string(g);
            t.MemoryInGb = 8 * (1 + (int)(rng() % 12)); t.VCPU = 4 * (int)(rng() % 9); t.RAMGb = 16 * (int)(rng() % 9);
            t.SecureCloud = rng() % 4 != 0; t.CommunityCloud = rng() % 3 != 0;
            t.SecurePrice = (double)(rng() % 200) / 100.0; t.CommunityPrice = (double)(rng() % 150) / 100.0;
            api->types.push_back(t);
        }
        prov.NotifyPods([this](const PodPtr& p) { notes.push_back(p->name + ":" + p->status.phase); });
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
    // what a reference select (PrepareColumnsBatch + rpk_select) offers each pending pod
    std::map<std::string, Ids> Reference() {
        std::vector<std::string> pending;
        std::vector<PodPtr> pods;
        for (const auto& n : names) {
            PodPtr p = prov.GetPod("default", n).first;
            if (p->status.phase == "Pending" && !p->annotations.count(PodIDAnnotation)) { pending.push_back(n); pods.push_back(p); }
        }
        std::map<std::string, Ids> want;
        const uint32_t P = (uint32_t)pods.size();
        if (P == 0) return want;
        PodColumnsSoA cols;
        PrepareColumnsBatch(pods, &cols);
        std::vector<GPUType> types;
        { std::lock_guard<std::mutex> g(api->mu); types = api->types; }
        std::vector<int32_t> mem, vcpu, ram, best(P), top5((size_t)P * RPK_TOPK);
        std::vector<double> sp, cp;
        std::vector<uint8_t> fl;
        for (const auto& t : types) {
            mem.push_back(t.MemoryInGb); vcpu.push_back(t.VCPU); ram.push_back(t.RAMGb); sp.push_back(t.SecurePrice); cp.push_back(t.CommunityPrice);
            fl.push_back((uint8_t)((t.SecureCloud ? RPK_FLAG_SECURE_CLOUD : 0u) | (t.CommunityCloud ? RPK_FLAG_COMMUNITY_CLOUD : 0u)));
        }
        rpk_ctx* ref = nullptr;
        CHECK_EQ(rpk_create(1, nullptr, &ref), RPK_OK);
        CHECK_EQ(rpk_offers_upload(ref, (uint32_t)types.size(), mem.data(), vcpu.data(), ram.data(), sp.data(), cp.data(), fl.data()), RPK_OK);
        CHECK_EQ(rpk_select(ref, P, cols.req_mem_gb.data(), cols.req_vcpu.data(), cols.req_ram_gb.data(), cols.max_price.data(),
                            cols.cloud.data(), best.data(), top5.data()), RPK_OK);
        rpk_destroy(ref);
        for (uint32_t i = 0; i < P; ++i) {
            Ids& w = want[pending[i]];
            for (int k = 0; k < RPK_TOPK; ++k) { const int32_t g = top5[(size_t)i * RPK_TOPK + k]; if (g >= 0) w.push_back(types[(size_t)g].ID); }
        }
        return want;
    }
};

// one round on a World: creates, a checked pending tick, a steady tick, churn, status changes and a sweep.  Returns the
// pods the round created.
static int Round(World& w, int round, int next, int creates) {
    for (int i = 0; i < creates; ++i) {
        const std::string n = "r" + std::to_string(next + i);
        w.names.insert(n);
        try { w.prov.CreatePod(w.Random(n)); } catch (const std::exception& e) { std::printf("FAIL CreatePod threw: %s\n", e.what()); ++g_fail; }
    }
    const std::map<std::string, Ids> want = w.Reference();
    w.api->ids_of.clear();
    const uint64_t rows = w.prov.ReselectedRows();
    w.prov.ProcessPendingPods();
    CHECK(w.api->ids_of == want);
    CHECK(w.prov.ReselectedRows() - rows <= want.size());  // only rows that are new or changed since the last tick
    const uint64_t rows2 = w.prov.ReselectedRows();
    w.api->ids_of.clear();
    w.prov.ProcessPendingPods();
    CHECK_EQ(w.prov.ReselectedRows(), rows2);  // a steady tick recomputes nothing, across the growth too
    CHECK(w.api->ids_of == want);
    w.api->refuses = [round](const std::string& n) { return std::stoi(n.substr(1)) % 7 != round % 7; };
    w.prov.ProcessPendingPods();
    w.api->refuses = [](const std::string&) { return true; };
    for (int k = 0; k < 40 && !w.names.empty(); ++k) {  // updates and deletes of random pods
        auto it = w.names.begin();
        std::advance(it, w.rng() % w.names.size());
        PodPtr cur = w.prov.GetPod("default", *it).first;
        if (k % 4 == 0) { w.prov.DeletePod(cur); w.names.erase(it); continue; }
        PodPtr up = w.Random(*it);
        if (cur->annotations.count(PodIDAnnotation)) up->annotations[PodIDAnnotation] = cur->annotations.at(PodIDAnnotation);
        w.prov.UpdatePod(up);
    }
    {
        static const char* sts[] = {"RUNNING", "EXITED", "RUNNING", "TERMINATED"};
        std::lock_guard<std::mutex> g(w.api->mu);
        int k = 0;
        for (auto& kv : w.api->status) if (k++ % 5 == round % 5) kv.second = sts[(k + round) % 4];
    }
    w.prov.UpdateAllPodStatuses();
    return creates;
}

static void TestGrowthMatchesALargeProvider() {
    World small(16), large(8192);
    int next = 0;
    for (int round = 0; next < 5000; ++round) {
        const int creates = round < 8 ? 3 + round * 5 : 400;
        Round(small, round, next, creates);
        Round(large, round, next, creates);
        next += creates;
        CHECK(small.api->ids_of == large.api->ids_of);
        CHECK_EQ(small.api->deploys, large.api->deploys);
        CHECK_EQ(small.prov.ReselectedRows(), large.prov.ReselectedRows());  // growth itself reselects no row
    }
    CHECK(small.notes == large.notes);  // every transition notified as often, in the same order, as without growth
    CHECK(!small.notes.empty());
    std::printf("growth: %zu notifications, %d deploys, %llu rows reselected\n", small.notes.size(), small.api->deploys,
                (unsigned long long)small.prov.ReselectedRows());
}

// one thread creates and deletes pods while another sweeps, across several growths: every RUNNING transition of the
// tracked pods is notified exactly once (the pattern of host_test.cc's concurrent test)
static void TestConcurrentCreateAndSweepAcrossGrowths() {
    auto api = std::make_shared<FakeRunPod>();
    GPUType t; t.ID = "gpu0"; t.MemoryInGb = 80; t.SecureCloud = true; t.SecurePrice = 0.2; t.CommunityPrice = 0.2;
    api->types.push_back(t);
    api->refuses = [](const std::string&) { return false; };
    Provider prov(api, 1, 16);
    std::mutex m;
    std::map<std::string, int> running_seen;
    prov.NotifyPods([&](const PodPtr& p) { if (p->status.phase == "Running") { std::lock_guard<std::mutex> g(m); ++running_seen[p->name]; } });
    for (int i = 0; i < 12; ++i) prov.CreatePod(MakePod("t" + std::to_string(i)));
    prov.UpdateAllPodStatuses();
    std::atomic<bool> stop{false};
    std::atomic<int> threw{0};
    std::thread churn([&] {  // 16 -> 32 -> ... -> 2048 slots while the sweeps run
        int k = 0;
        while (!stop) {
            try {
                prov.CreatePod(MakePod("churn" + std::to_string(k)));
                if (k % 3 == 0) prov.DeletePod(prov.GetPod("default", "churn" + std::to_string(k)).first);
            } catch (...) { ++threw; }
            if (++k == 1500) break;
        }
    });
    for (int round = 0; round < 12; ++round) {
        api->SetStatus("rp-" + std::to_string(round + 1), "RUNNING");
        prov.UpdateAllPodStatuses();
    }
    churn.join();
    stop = true;
    prov.UpdateAllPodStatuses();
    CHECK_EQ(threw.load(), 0);
    for (int i = 0; i < 12; ++i) { std::lock_guard<std::mutex> g(m); CHECK_EQ(running_seen["t" + std::to_string(i)], 1); }
}

int main() {
    TestGrowthMatchesALargeProvider();
    TestConcurrentCreateAndSweepAcrossGrowths();
    std::printf("%s: %d checks, %d failed (gpu)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
