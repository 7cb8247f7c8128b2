// host_slots_test.cc -- the Provider's status sweep diffs only the slots it fetched this cycle (rpk_status_diff_slots):
// pods the reference skips before its compare -- terminal phase (kubelet.go:836), no RunPod id (:841-844), failed fetch
// (:848-855), NOT_FOUND (:861-864) -- are not uploaded, and the engine's status_records grows by the fetched pods only.
// Needs a GPU (the Provider refuses to start without one).
#include <cstdio>
#include <mutex>
#include <set>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

struct ScriptedRunPod : RunPodAPI {
    std::mutex mu;
    std::map<std::string, DetailedStatus> status;
    bool fail_deploy = false;
    int deploys = 0;
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string*) override {
        *out = {{"A4000", "", 16, true, .32, true, .17}, {"A40", "", 48, true, .40, false, 0}};
        return true;
    }
    bool DeployPod(const Pod&, const std::vector<std::string>& ids, int, const std::string&, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        if (fail_deploy || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
        status[*id] = {"STARTING", {}};
        return true;
    }
    bool GetDetailedPodStatus(const std::string& id, DetailedStatus* out, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        auto it = status.find(id);
        if (it == status.end()) { *err = "http 500"; return false; }
        *out = it->second; return true;
    }
    bool TerminatePod(const std::string&, std::string*) override { return true; }
};

static PodPtr MakePod(const std::string& name) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->status.phase = "Pending";
    return p;
}

static uint64_t StatusRecords(Provider& prov) {
    rpk_stats st;
    rpk_stats_get(prov.Ctx(), &st);
    return st.status_records;
}

static void TestSweepDiffsFetchedSlotsOnly() {
    auto api = std::make_shared<ScriptedRunPod>();
    Provider prov(api, 1, 512);
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase); });
    for (int i = 0; i < 12; ++i) prov.CreatePod(MakePod("s" + std::to_string(i)));  // s0..s11 = rp-1..rp-12
    api->fail_deploy = true;
    for (int i = 0; i < 3; ++i) prov.CreatePod(MakePod("noid" + std::to_string(i)));  // tracked, never deployed: no RunPod id
    api->fail_deploy = false;

    uint64_t rec = StatusRecords(prov);
    prov.UpdateAllPodStatuses();  // the 12 deployed pods are fetched; the 3 without an id are skipped
    CHECK_EQ(StatusRecords(prov) - rec, 12u);
    CHECK_EQ(notified.size(), 12u);  // no ports requested: exposed, while CreatePod stored "not exposed"
    notified.clear();

    api->status["rp-1"].DesiredStatus = "EXITED";
    api->status["rp-2"].DesiredStatus = "TERMINATED";
    rec = StatusRecords(prov);
    prov.UpdateAllPodStatuses();
    CHECK_EQ(StatusRecords(prov) - rec, 12u);
    CHECK_EQ(notified.size(), 2u);  // s0, s1 -> Succeeded: terminal from now on
    notified.clear();

    api->status.erase("rp-3");                       // s2: fetch fails this cycle
    api->status["rp-4"].DesiredStatus = "NOT_FOUND"; // s3: diverted to handleMissingRunPodInstance
    api->status["rp-5"].DesiredStatus = "RUNNING";   // s4: a change among the listed slots
    rec = StatusRecords(prov);
    prov.UpdateAllPodStatuses();
    CHECK_EQ(StatusRecords(prov) - rec, 12u - 2u - 1u - 1u);
    std::set<std::string> s(notified.begin(), notified.end());
    CHECK_EQ(notified.size(), 2u); CHECK_EQ(s.count("s4:Running"), 1u); CHECK_EQ(s.count("s3:Failed"), 1u);
    notified.clear();

    api->status["rp-3"] = {"RUNNING", {}};  // s2 is fetched again and reports its change; s3 has no id any more
    rec = StatusRecords(prov);
    prov.UpdateAllPodStatuses();
    CHECK_EQ(StatusRecords(prov) - rec, 12u - 2u - 1u);
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified.empty() ? "" : notified[0], "s2:Running");
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 0u);
}

int main() {
    TestSweepDiffsFetchedSlotsOnly();
    std::printf("%s: %d checks, %d failed (gpu)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
