// host_explain_test.cc -- Provider::ExplainUnschedulable on the ten offers of SURVEY.md 8(c).  A Provider with a scripted
// fake API gets a mix of pods: some fit, some fit no GPU type for a memory, price, cloud or vCPU request.  After one
// pending tick the call lists exactly the pods whose gpuTypeIds list came back empty, ascending by slot, with the
// pinned messages; a pod whose annotation is fixed deploys on the next tick and drops out, and pods failed after 15
// minutes are not listed, though the tick that failed them left their flags and empty lists behind; and the deploys and
// notifications equal those of a Provider that never calls it.  Then a random mix of 400 pods over a 300-offer table
// checks every explanation against rpk_explain on the pod's columns.  Needs a GPU (the Provider refuses to start
// without one).
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <random>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

using Ids = std::vector<std::string>;

struct FakeRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;
    int deploys = 0;
    std::vector<std::string> log;  // "name:id,id,..." per deploy attempt, in order
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string*) override {
        std::lock_guard<std::mutex> g(mu);
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const Ids& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        std::string e = pod.name + ":";
        for (const auto& s : ids) e += s + ",";
        log.push_back(e);
        if (ids.empty()) { *err = "no GPU type"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
        return true;
    }
    bool GetDetailedPodStatus(const std::string&, DetailedStatus* out, std::string*) override { out->DesiredStatus = "RUNNING"; return true; }
    bool TerminatePod(const std::string&, std::string*) override { return true; }
};

static GPUType Type(const char* id, int mem, bool s, double sp, bool c, double cp) {
    GPUType t;
    t.ID = id; t.DisplayName = id; t.MemoryInGb = mem; t.SecureCloud = s; t.SecurePrice = sp; t.CommunityCloud = c; t.CommunityPrice = cp;
    return t;
}

static std::vector<GPUType> KatTable() {
    return {Type("A4000", 16, true, .32, true, .17), Type("A5000", 24, true, .36, true, .22), Type("RTX3090", 24, false, 0, true, .22),
            Type("A40", 48, true, .40, false, 0), Type("RTX4090", 24, true, .69, true, .34), Type("L4", 24, true, .43, false, 0),
            Type("A100", 80, true, 1.64, true, 1.19), Type("T4free", 16, true, 0, true, 0), Type("A4500", 20, true, .34, true, .19),
            Type("edge", 32, true, .5, true, .5)};
}

static PodPtr MakePod(const std::string& name, Annotations ann = {}) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending"; p->annotations = std::move(ann);
    return p;
}

struct World {
    std::shared_ptr<FakeRunPod> api = std::make_shared<FakeRunPod>();
    std::vector<std::string> notes;
    Provider prov;
    bool explain;
    World(bool explain_each_tick) : prov(api, 1, 64), explain(explain_each_tick) {
        api->types = KatTable();
        prov.NotifyPods([this](const PodPtr& p) { notes.push_back(p->name + ":" + p->status.phase); });
    }
    std::vector<Unschedulable> Tick() {
        prov.ProcessPendingPods();
        return explain ? prov.ExplainUnschedulable() : std::vector<Unschedulable>();
    }
};

static void Populate(World& w) {
    w.prov.CreatePod(MakePod("fits"));                                                           // 16 GB, $0.50, SECURE
    w.prov.CreatePod(MakePod("big", {{GpuMemoryAnnotation, "80"}}));                             // KAT row 1
    w.prov.CreatePod(MakePod("cheap", {{GpuMemoryAnnotation, "24"}, {MaxPriceAnnotation, "0.2"}, {CloudTypeAnnotation, "COMMUNITY"}}));
    w.prov.CreatePod(MakePod("cpus", {{VcpuAnnotation, "64"}}));                                // the table has no vCPUs
    w.prov.CreatePod(MakePod("fits2", {{GpuMemoryAnnotation, "24"}, {CloudTypeAnnotation, "COMMUNITY"}}));
}

static const char* kBig = "0/10 GPU types fit: 2 not offered in SECURE cloud, 3 at or above $0.50/hr, 7 under 80 GB GPU memory. "
                          "Nearest: A100 needs a max price above $1.64/hr; A4000 has 16 GB GPU memory.";
static const char* kCheap = "0/10 GPU types fit: 3 not offered in COMMUNITY cloud, 5 at or above $0.20/hr, 2 under 24 GB GPU memory. "
                            "Nearest: A5000 needs a max price above $0.22/hr; A4000 has 16 GB GPU memory.";
static const char* kCpus = "0/10 GPU types fit: 2 not offered in SECURE cloud, 3 at or above $0.50/hr, 8 under 64 vCPUs. "
                           "Nearest: A4000 has 0 vCPUs.";

static void KnownAnswers() {
    World with(true), without(false);
    Populate(with); Populate(without);
    CHECK(with.prov.ExplainUnschedulable().empty());  // no pending tick yet: nothing is flagged
    const std::vector<Unschedulable> u = with.Tick();
    without.Tick();
    CHECK_EQ(u.size(), (size_t)3);
    if (u.size() == 3) {
        CHECK_EQ(u[0].name, std::string("big")); CHECK_EQ(u[0].message, std::string(kBig));
        CHECK_EQ(u[1].name, std::string("cheap")); CHECK_EQ(u[1].message, std::string(kCheap));
        CHECK_EQ(u[2].name, std::string("cpus")); CHECK_EQ(u[2].message, std::string(kCpus));
        CHECK_EQ(u[0].ns, std::string("default"));
        CHECK_EQ(u[0].why.n_feasible, 0u); CHECK_EQ(u[0].why.n_unoffered, 2u);
        CHECK_EQ(u[0].why.n_only[RPK_REQ_PRICE], 1u); CHECK_EQ(u[0].why.n_only[RPK_REQ_MEM], 5u);
        CHECK_EQ(u[0].why.nearest[RPK_REQ_PRICE], 6); CHECK_EQ(u[0].why.nearest[RPK_REQ_MEM], 0);
        CHECK_EQ(u[0].why.nearest[RPK_REQ_VCPU], -1); CHECK_EQ(u[0].why.nearest[RPK_REQ_RAM], -1);
    }
    for (const auto& x : with.prov.ExplainUnschedulable()) CHECK(x.name != "fits" && x.name != "fits2");
    // fix "big": the next tick deploys it, and it drops out
    for (World* w : {&with, &without}) w->prov.UpdatePod(MakePod("big", {{GpuMemoryAnnotation, "48"}}));
    const std::vector<Unschedulable> u2 = with.Tick();
    without.Tick();
    CHECK_EQ(u2.size(), (size_t)2);
    for (const auto& x : u2) CHECK(x.name != "big");
    CHECK(with.prov.GetPod("default", "big").first->annotations.count(PodIDAnnotation) == 1);
    // the sweeps and a third tick, and everything either Provider did is the same
    for (World* w : {&with, &without}) { w->prov.UpdateAllPodStatuses(); w->prov.SetClock(16 * 60); }
    // this tick fails the pods that never fit (15 minutes): the flags and lists still name them, but none is pending
    CHECK(with.Tick().empty());
    without.Tick();
    CHECK(with.prov.ExplainUnschedulable().empty());
    CHECK(with.api->log == without.api->log);
    CHECK(with.notes == without.notes);
    CHECK_EQ(with.prov.SelectCalls(), without.prov.SelectCalls());
    CHECK_EQ(with.prov.ReselectedRows(), without.prov.ReselectedRows());
    CHECK(!with.notes.empty());  // the 15-minute failure of the pods that never fit
    for (const char* n : {"big", "cheap", "cpus", "fits", "fits2"}) {
        const auto a = with.prov.GetPodStatus("default", n), b = without.prov.GetPodStatus("default", n);
        CHECK_EQ(a.first.phase, b.first.phase);
        CHECK_EQ(a.first.message, b.first.message);
    }
}

// 400 random pods on a 300-offer table: every explanation equals rpk_explain of the pod's columns, and the list holds
// exactly the pods whose deploy got no GPU type
static void RandomMix() {
    std::mt19937 rng(7);
    World w(true);
    w.api->types.clear();
    for (int g = 0; g < 300; ++g) {
        GPUType t = Type("", 8 * (1 + (int)(rng() % 12)), rng() % 4 != 0, (double)(rng() % 200) / 100.0, rng() % 3 != 0, (double)(rng() % 150) / 100.0);
        t.ID = "gpu" + std::to_string(g); t.VCPU = 4 * (int)(rng() % 9); t.RAMGb = 16 * (int)(rng() % 9);
        w.api->types.push_back(t);
    }
    static const char* mems[] = {"", "16", "48", "96", "200"};
    static const char* prices[] = {"", "0.05", "0.5", "1.5"};
    std::vector<PodPtr> pods;
    for (int i = 0; i < 400; ++i) {
        Annotations a{{GpuMemoryAnnotation, mems[rng() % 5]}, {MaxPriceAnnotation, prices[rng() % 4]}};
        if (rng() % 2) a[CloudTypeAnnotation] = "COMMUNITY";
        if (rng() % 3 == 0) a[VcpuAnnotation] = std::to_string(8 * (rng() % 8));
        if (rng() % 3 == 0) a[RamAnnotation] = std::to_string(32 * (rng() % 8));
        pods.push_back(MakePod("m" + std::to_string(i), a));
        w.prov.CreatePod(pods.back());
    }
    w.api->log.clear();
    const std::vector<Unschedulable> u = w.Tick();
    std::map<std::string, bool> empty_deploy;
    for (const auto& e : w.api->log) empty_deploy[e.substr(0, e.find(':'))] = e.back() == ':';
    size_t n_empty = 0;
    for (const auto& kv : empty_deploy) n_empty += kv.second;
    CHECK_EQ(u.size(), n_empty);
    CHECK(n_empty > 20 && n_empty < 380);
    rpk_ctx* ref = nullptr;
    CHECK_EQ(rpk_create(1, nullptr, &ref), RPK_OK);
    std::vector<int32_t> mem, vcpu, ram;
    std::vector<double> sp, cp;
    std::vector<uint8_t> fl;
    for (const auto& t : w.api->types) {
        mem.push_back(t.MemoryInGb); vcpu.push_back(t.VCPU); ram.push_back(t.RAMGb); sp.push_back(t.SecurePrice); cp.push_back(t.CommunityPrice);
        fl.push_back((uint8_t)((t.SecureCloud ? RPK_FLAG_SECURE_CLOUD : 0u) | (t.CommunityCloud ? RPK_FLAG_COMMUNITY_CLOUD : 0u)));
    }
    CHECK_EQ(rpk_offers_upload(ref, (uint32_t)mem.size(), mem.data(), vcpu.data(), ram.data(), sp.data(), cp.data(), fl.data()), RPK_OK);
    for (const auto& x : u) {
        CHECK(empty_deploy[x.name]);
        const PodColumns c = PrepareColumns(*w.prov.GetPod(x.ns, x.name).first);
        rpk_explanation want;
        CHECK_EQ(rpk_explain(ref, 1, &c.req_mem_gb, &c.req_vcpu, &c.req_ram_gb, &c.max_price, &c.cloud, &want), RPK_OK);
        CHECK(std::memcmp(&want, &x.why, sizeof(want)) == 0);
        CHECK_EQ(x.why.n_feasible, 0u);
        CHECK_EQ(x.message, UnschedulableMessage(want, 300, c, w.api->types));
    }
    rpk_destroy(ref);
}

int main() {
    try {
        KnownAnswers();
        RandomMix();
    } catch (const std::exception& e) {
        std::printf("FAIL exception: %s\n", e.what());
        ++g_fail;
    }
    std::printf("ok: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
