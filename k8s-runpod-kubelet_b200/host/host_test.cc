// host_test.cc -- tests of the C++ Provider mirror, shaped like the reference's own tests
// (pkg/virtual_kubelet/annotations_test.go: build a pod (+ owner Job), prepare the RunPod parameters, assert
// minRAMPerGPU / cloudType / gpuTypeIds) plus the batched tick bodies.  `--cpu`: host logic only (no GPU).
// `--gpu`: the full Provider over the CUDA engine with a scripted RunPod API.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <cctype>
#include <cerrno>
#include <climits>
#include <cstdlib>
#include <atomic>
#include <mutex>
#include <set>
#include <thread>

#include "rpk_host.hpp"

using namespace rpkhost;

static int g_fail = 0, g_checks = 0;
#define CHECK(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); } } while (0)
#define CHECK_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d: %s == %s\n", __FILE__, __LINE__, #a, #b); } } while (0)

static PodPtr MakePod(const std::string& name, Annotations ann = {}, std::shared_ptr<Annotations> job = nullptr) {
    auto p = std::make_shared<Pod>();
    p->ns = "default"; p->name = name; p->annotations = std::move(ann); p->owner_job = std::move(job);
    p->status.phase = "Pending";
    return p;
}

// ---- host logic (no GPU) ---------------------------------------------------------------------------------
static void TestColumnProducers() {
    // annotations_test.go:84-90: job carries memory "8", cloud "SECURE"
    auto job = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "8"}, {CloudTypeAnnotation, "SECURE"},
                                                         {TemplateIdAnnotation, "tmpl"}, {ContainerRegistryAuthAnnotation, "auth"}});
    auto pod = MakePod("test-pod", {}, job);
    PodColumns c = PrepareColumns(*pod);
    CHECK_EQ(c.req_mem_gb, 8);             // annotations_test.go:117-118
    CHECK_EQ(c.cloud_type, "SECURE");      // :121-122
    CHECK_EQ(c.max_price, 0.5);            // runpod_client.go:1281 passes DefaultMaxPrice
    CHECK_EQ(c.req_vcpu, 0); CHECK_EQ(c.req_ram_gb, 0);
    CHECK_EQ(GetAnnotationWithFallback(*pod, TemplateIdAnnotation, ""), "tmpl");
    // :124-143 pod annotations override the job's
    auto pod2 = MakePod("p2", {{ContainerRegistryAuthAnnotation, "pod-auth-override"}, {GpuMemoryAnnotation, "16"}}, job);
    CHECK_EQ(PrepareColumns(*pod2).req_mem_gb, 16);
    CHECK_EQ(GetAnnotationWithFallback(*pod2, ContainerRegistryAuthAnnotation, ""), "pod-auth-override");
    CHECK_EQ(GetAnnotationWithFallback(*pod2, TemplateIdAnnotation, ""), "tmpl");
    // :186-234 job: COMMUNITY + "24"; pod overrides the cloud type with SECURE
    auto job2 = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "24"}, {CloudTypeAnnotation, "COMMUNITY"}, {DatacenterAnnotation, "US-TX-3"}});
    auto pod3 = MakePod("p3", {{CloudTypeAnnotation, "SECURE"}}, job2);
    CHECK_EQ(PrepareColumns(*pod3).req_mem_gb, 24);
    CHECK_EQ(PrepareColumns(*pod3).cloud_type, "SECURE");
    CHECK_EQ(PrepareColumns(*MakePod("p4", {}, job2)).cloud_type, "COMMUNITY");
    // runpod_test.go:89-90: "STANDARD" is invalid -> SECURE; memory "2"
    auto pod5 = MakePod("p5", {{CloudTypeAnnotation, "STANDARD"}, {GpuMemoryAnnotation, "2"}});
    CHECK_EQ(PrepareColumns(*pod5).cloud_type, "SECURE");
    CHECK_EQ(PrepareColumns(*pod5).req_mem_gb, 2);
    // extractGPUMemory / validateCloudType corner cases (runpod_client.go:1115-1134, 1181-1191)
    CHECK_EQ(ExtractGPUMemory(""), 16); CHECK_EQ(ExtractGPUMemory("abc"), 16); CHECK_EQ(ExtractGPUMemory("24GB"), 16);
    CHECK_EQ(ExtractGPUMemory(" 8"), 16); CHECK_EQ(ExtractGPUMemory("+8"), 8); CHECK_EQ(ExtractGPUMemory("-4"), -4);
    CHECK_EQ(ExtractGPUMemory("9223372036854775808"), 16); CHECK_EQ(ExtractGPUMemory("1_6"), 16);
    CHECK_EQ(PrepareColumns(*MakePod("big", {{GpuMemoryAnnotation, "99999999999"}})).req_mem_gb, INT32_MAX);
    CHECK_EQ(ValidateCloudType("community"), "COMMUNITY"); CHECK_EQ(ValidateCloudType(" SECURE"), "SECURE");
    CHECK_EQ(ValidateCloudType("commun\xC4\xB1ty"), "COMMUNITY"); CHECK_EQ(ValidateCloudType("ALL"), "SECURE");
    // extension annotations
    auto ext = MakePod("ext", {{MaxPriceAnnotation, "1.25"}, {VcpuAnnotation, "16"}, {RamAnnotation, "64"}});
    CHECK_EQ(PrepareColumns(*ext).max_price, 1.25); CHECK_EQ(PrepareColumns(*ext).req_vcpu, 16); CHECK_EQ(PrepareColumns(*ext).req_ram_gb, 64);
    CHECK_EQ(PrepareColumns(*MakePod("bad", {{MaxPriceAnnotation, "cheap"}})).max_price, 0.5);
}

static void TestPortsAndTranslate() {
    // GetRequestedPorts: annotation override, comma separated, trimmed (runpod_client.go:1381-1393)
    auto p = MakePod("ports", {{PortsAnnotation, "8080/http, 5432/tcp ,22/tcp"}});
    p->container_ports = {"9999/tcp"};
    auto rp = GetRequestedPorts(*p);
    CHECK_EQ(rp.size(), 3u); CHECK_EQ(rp[1], "5432/tcp"); CHECK_EQ(rp[2], "22/tcp");
    p->annotations.clear();
    CHECK_EQ(GetRequestedPorts(*p)[0], "9999/tcp");
    // checkPortsExposed (kubelet.go:566-605)
    CHECK(CheckPortsExposed({}, {}));
    CHECK(CheckPortsExposed({{"5432", 30001}}, {"5432/tcp"}));
    CHECK(!CheckPortsExposed({}, {"5432/tcp"}));
    CHECK(CheckPortsExposed({}, {"8080/http"}));                       // HTTP assumed proxied
    CHECK(!CheckPortsExposed({{"8080", 1}}, {"8080/http", "22/tcp"}));
    CHECK(CheckPortsExposed({{"22", 1}}, {"8080/http", "22/tcp"}));
    // translateRunPodStatus (kubelet.go:1848-2024)
    auto v = TranslateRunPodStatus("RUNNING", "", true);
    CHECK_EQ(v.phase, "Running"); CHECK(v.ready); CHECK(v.started); CHECK_EQ(v.state, "Running");
    v = TranslateRunPodStatus("RUNNING", "", false);
    CHECK_EQ(v.phase, "Pending"); CHECK(!v.ready); CHECK_EQ(v.reason, "ContainerCreating");
    v = TranslateRunPodStatus("STARTING", "pulling", true);
    CHECK_EQ(v.phase, "Pending"); CHECK_EQ(v.state, "Waiting"); CHECK_EQ(v.message, "pulling");
    v = TranslateRunPodStatus("EXITED", "done", true);
    CHECK_EQ(v.phase, "Succeeded"); CHECK_EQ(v.reason, "Completed"); CHECK_EQ(v.exit_code, 0);
    v = TranslateRunPodStatus("EXITED", "Container FAILED to start", true);
    CHECK_EQ(v.phase, "Failed"); CHECK_EQ(v.reason, "Error"); CHECK_EQ(v.exit_code, 1);
    v = TranslateRunPodStatus("TERMINATING", "", false);
    CHECK_EQ(v.phase, "Running"); CHECK(v.ready);
    v = TranslateRunPodStatus("TERMINATED", "", true);
    CHECK_EQ(v.phase, "Succeeded"); CHECK_EQ(v.reason, "Terminated");
    v = TranslateRunPodStatus("NOT_FOUND", "", true);
    CHECK_EQ(v.phase, "Failed"); CHECK_EQ(v.reason, "PodDeleted"); CHECK_EQ(v.exit_code, 1);
    v = TranslateRunPodStatus("PAUSED", "", true);
    CHECK_EQ(v.phase, "Unknown"); CHECK_EQ(v.reason, "ContainerStatusUnknown"); CHECK(!v.ready);
    // record slot
    CHECK_EQ(TranslateRunPodStatus("RUNNING", "m", false).container_message, "Container reported as running but ports not yet exposed");  // :1885
    CHECK_EQ(TranslateRunPodStatus("NOT_FOUND", "m", true).container_message, "Pod was deleted from RunPod API");                            // :1963
    CHECK_EQ(TranslateRunPodStatus("PAUSED", "m", true).container_message, "Unknown RunPod status: PAUSED");                                // :1975
    CHECK_EQ(TranslateRunPodStatus("EXITED", "oom", true).container_message, "oom"); CHECK_EQ(TranslateRunPodStatus("RUNNING", "m", true).container_message, "");
    // the kernel's code -> the same view (codes as documented in include/rpk.h; the GPU tests pin the kernel to them)
    struct { const char* status; const char* msg; bool ports; uint16_t code; } kCodes[] = {
        {"RUNNING", "", true, 0x003A}, {"RUNNING", "x", false, 0x0901}, {"STARTING", "pulling", true, 0x0101}, {"EXITED", "done", true, 0x0243},
        {"EXITED", "it FAILED", false, 0x03C4}, {"TERMINATING", "", false, 0x003A}, {"TERMINATED", "bye", true, 0x0443},
        {"NOT_FOUND", "", true, 0x15C4}, {"PAUSED", "", false, 0x1E00}};
    for (auto& k : kCodes) CHECK(StatusFromCode(k.code, k.status, k.msg) == TranslateRunPodStatus(k.status, k.msg, k.ports));
    CHECK(MessageHasError("Some ERROR")); CHECK(MessageHasError("it Failed")); CHECK(!MessageHasError("fine"));
    // record slot
    uint8_t slot[32];
    CHECK(EncodeStatusRecord(slot, 32, "RUNNING", true));
    CHECK_EQ(slot[0], 9); CHECK(std::memcmp(slot + 1, "RUNNING", 7) == 0); CHECK_EQ(slot[8], 0); CHECK_EQ(slot[9], 1); CHECK_EQ(slot[10], 0);
    CHECK(EncodeStatusRecord(slot, 16, "TERMINATING", true, true));  // every RunPod status fits the 16-byte slot
    CHECK_EQ(slot[0], 13 | 0x80); CHECK_EQ(slot[13], 1);
    CHECK(!EncodeStatusRecord(slot, 16, "TERMINATINGXYZ", false));
    CHECK(!EncodeStatusRecord(slot, 32, std::string(30, 'x'), false));
}

// ---- scripted RunPod API -----------------------------------------------------------------------------------
struct FakeRunPod : RunPodAPI {
    std::vector<GPUType> types;
    std::mutex mu;  // the threaded tests call the API from several threads
    std::map<std::string, DetailedStatus> status;
    void SetStatus(const std::string& id, const std::string& st) { std::lock_guard<std::mutex> g(mu); status[id].DesiredStatus = st; }
    bool fail_deploy = false, fail_fetch = false;
    int fetches = 0, deploys = 0, terminated = 0, status_gets = 0;
    struct Call { std::string pod; std::vector<std::string> ids; int min_ram; std::string cloud; };
    std::vector<Call> calls;
    bool FetchGPUTypes(std::vector<GPUType>* out, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        ++fetches;
        if (fail_fetch) { *err = "graphql down"; return false; }
        *out = types; return true;
    }
    bool DeployPod(const Pod& pod, const std::vector<std::string>& ids, int min_ram, const std::string& cloud, std::string* id, double* cost, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        calls.push_back({pod.name, ids, min_ram, cloud});
        if (fail_deploy || ids.empty()) { *err = "no capacity"; return false; }
        *id = "rp-" + std::to_string(++deploys); *cost = 0.25;
        status[*id] = {"STARTING", {}};
        return true;
    }
    bool GetDetailedPodStatus(const std::string& id, DetailedStatus* out, std::string* err) override {
        std::lock_guard<std::mutex> g(mu);
        ++status_gets;
        auto it = status.find(id);
        if (it == status.end()) { *err = "http 500"; return false; }
        *out = it->second; return true;
    }
    bool TerminatePod(const std::string&, std::string*) override { std::lock_guard<std::mutex> g(mu); ++terminated; return true; }
};

static std::vector<GPUType> KatTable() {  // tests/golden/select_kat.json (SURVEY.md 8c)
    return {{"A4000", "", 16, true, .32, true, .17}, {"A5000", "", 24, true, .36, true, .22}, {"RTX3090", "", 24, false, 0, true, .22},
            {"A40", "", 48, true, .40, false, 0},    {"RTX4090", "", 24, true, .69, true, .34}, {"L4", "", 24, true, .43, false, 0},
            {"A100", "", 80, true, 1.64, true, 1.19}, {"T4free", "", 16, true, 0, true, 0},     {"A4500", "", 20, true, .34, true, .19},
            {"edge", "", 32, true, .5, true, .5}};
}

static void TestProviderDeployPath() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 256);
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase); });
    // annotations_test.go scenario 1: job annotations -> minRAMPerGPU 8, SECURE
    auto job = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "8"}, {CloudTypeAnnotation, "SECURE"}});
    CHECK_EQ(prov.CreatePod(MakePod("a", {}, job)), "");
    CHECK_EQ(api->calls.back().min_ram, 8); CHECK_EQ(api->calls.back().cloud, "SECURE");
    CHECK_EQ(api->calls.back().ids, (std::vector<std::string>{"A4000", "A4500", "A5000", "A40", "L4"}));  // KAT (16|8, .5, SECURE)
    // scenario 2: pod overrides job -> 16
    prov.CreatePod(MakePod("b", {{GpuMemoryAnnotation, "16"}}, job));
    CHECK_EQ(api->calls.back().min_ram, 16);
    // scenario 3: job 24 + COMMUNITY, pod says SECURE -> 24, SECURE -> [A5000, A40, L4]
    auto job2 = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "24"}, {CloudTypeAnnotation, "COMMUNITY"}});
    prov.CreatePod(MakePod("c", {{CloudTypeAnnotation, "SECURE"}}, job2));
    CHECK_EQ(api->calls.back().ids, (std::vector<std::string>{"A5000", "A40", "L4"}));
    prov.CreatePod(MakePod("d", {}, job2));  // COMMUNITY: tie 0.22 -> lower index first
    CHECK_EQ(api->calls.back().ids, (std::vector<std::string>{"A5000", "RTX3090", "RTX4090"}));
    // the table was uploaded once although it was fetched per call
    CHECK_EQ(prov.OfferUploads(), 1u); CHECK_EQ(api->fetches, 4);
    // deployed pods carry the two write-back annotations (kubelet.go:523-524)
    auto got = prov.GetPod("default", "a");
    CHECK(got.second.empty()); CHECK_EQ(got.first->annotations.at(PodIDAnnotation), "rp-1");
    CHECK(got.first->annotations.count(CostAnnotation) == 1);
    // unknown keys: error strings of kubelet.go:663, 680
    CHECK_EQ(prov.GetPod("default", "zz").second, "pod default-zz not found");
    CHECK_EQ(prov.GetPodStatus("default", "zz").second, "pod status not found for default-zz");
    CHECK_EQ(prov.GetPods().size(), 4u);

    // ---- batched retry: 40 pods whose deploy fails at CreatePod (swallowed), then one tick ----
    api->fail_deploy = true;
    for (int i = 0; i < 40; ++i) CHECK_EQ(prov.CreatePod(MakePod("pend" + std::to_string(i), {{GpuMemoryAnnotation, i % 2 ? "24" : "48"}})), "");
    const uint64_t sel_before = prov.SelectCalls();
    const int fetch_before = api->fetches;
    api->fail_deploy = false;
    api->calls.clear();
    prov.ProcessPendingPods();
    CHECK_EQ(prov.SelectCalls(), sel_before + 1);   // ONE rpk_select for the whole batch
    CHECK_EQ(api->fetches, fetch_before + 1);       // ONE GraphQL fetch per tick (reference: one per pod)
    CHECK_EQ(api->calls.size(), 40u);
    for (auto& c : api->calls) CHECK_EQ(c.ids, c.min_ram == 24 ? (std::vector<std::string>{"A5000", "A40", "L4"}) : (std::vector<std::string>{"A40"}));
    prov.ProcessPendingPods();                      // everything has a pod-id now: nothing to do
    CHECK_EQ(prov.SelectCalls(), sel_before + 1);
    // a pod nothing can satisfy: retried every tick, Failed + notified after 15 minutes (kubelet.go:786-810)
    prov.SetClock(1000);
    prov.CreatePod(MakePod("huge", {{GpuMemoryAnnotation, "640"}}));
    prov.ProcessPendingPods();
    CHECK(notified.empty());
    prov.SetClock(1000 + 15 * 60 + 1);
    prov.ProcessPendingPods();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "huge:Failed");
    CHECK_EQ(prov.GetPod("default", "huge").first->status.reason, "RunPodDeploymentFailed");
    // GraphQL outage: deploy step fails, CreatePod still returns nil and tracks the pod
    api->fail_fetch = true;
    CHECK_EQ(prov.CreatePod(MakePod("outage")), "");
    CHECK(prov.GetPod("default", "outage").first != nullptr);
    api->fail_fetch = false;
    // DeletePod: terminate + untrack (kubelet.go:621-651)
    auto a = prov.GetPod("default", "a").first;
    prov.DeletePod(a);
    CHECK_EQ(api->terminated, 1); CHECK(prov.GetPod("default", "a").first == nullptr);
}

static void TestProviderStatusSweep() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 128);
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase + (p->status.ready ? ":ready" : "")); });
    for (int i = 0; i < 20; ++i) {
        auto p = MakePod("w" + std::to_string(i), i % 2 ? Annotations{{PortsAnnotation, "5432/tcp"}} : Annotations{});
        prov.CreatePod(p);
    }
    // sweep 1: every instance is still STARTING.  Pods that requested no ports count as "exposed"
    // (kubelet.go:568-570) while CreatePod stored PortsExposed=false (:399), so exactly those ten report a
    // portsExposureChanged on the first sweep -- the reference does the same; the others are unchanged.
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 10u); CHECK_EQ(prov.StatusCalls(), 1u); CHECK_EQ(api->status_gets, 20);
    for (auto& n : notified) CHECK(n.size() > 8 && n.substr(n.size() - 8) == ":Pending" && std::stoi(n.substr(1, n.find(':') - 1)) % 2 == 0);
    CHECK(prov.Info("default", "w0")->PortsExposed); CHECK(!prov.Info("default", "w1")->PortsExposed);
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
    // instances 1..10 go RUNNING; odd ones requested a TCP port that is not mapped yet
    for (int i = 1; i <= 10; ++i) api->status["rp-" + std::to_string(i)].DesiredStatus = "RUNNING";
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 10u);
    std::set<std::string> s(notified.begin(), notified.end());
    CHECK(s.count("w0:Running:ready") == 1);   // no ports requested -> exposed -> Running
    CHECK(s.count("w1:Pending") == 1);         // RUNNING but 5432/tcp not mapped -> Pending / ContainerCreating
    CHECK_EQ(prov.Info("default", "w1")->Status, "RUNNING"); CHECK(!prov.Info("default", "w1")->PortsExposed);
    // the port shows up: status string unchanged, portsExposureChanged alone triggers (kubelet.go:871)
    notified.clear();
    api->status["rp-2"].PortMappings["5432"] = 31000;  // rp-2 is w1
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "w1:Running:ready");
    // nothing moved: no callbacks
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
    // EXITED -> Succeeded (terminal: skipped by later sweeps, kubelet.go:836); unknown status -> Unknown
    api->status["rp-1"].DesiredStatus = "EXITED";
    api->status["rp-3"].DesiredStatus = "PAUSED";
    prov.UpdateAllPodStatuses();
    s = std::set<std::string>(notified.begin(), notified.end());
    CHECK_EQ(notified.size(), 2u); CHECK(s.count("w0:Succeeded") == 1); CHECK(s.count("w2:Unknown") == 1);
    const int gets = api->status_gets;
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty()); CHECK_EQ(api->status_gets, gets + 19);  // w0 is terminal now
    // a fetch error skips the pod for this cycle only (kubelet.go:848-855)
    api->status.erase("rp-5");
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
    // NOT_FOUND is diverted before the diff (kubelet.go:861-864): annotations dropped, pod Failed
    api->status["rp-6"].DesiredStatus = "NOT_FOUND";
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "w5:Failed");
    CHECK(prov.GetPod("default", "w5").first->annotations.count(PodIDAnnotation) == 0);
    CHECK_EQ(prov.Info("default", "w5")->Status, "EXITED");
    // GetPodStatus does its own live port check (kubelet.go:684-692)
    api->status["rp-4"].DesiredStatus = "RUNNING";  // w3 requested 5432/tcp
    prov.UpdateAllPodStatuses();
    CHECK_EQ(prov.GetPodStatus("default", "w3").first.phase, "Pending");
    api->status["rp-4"].PortMappings["5432"] = 1;
    CHECK_EQ(prov.GetPodStatus("default", "w3").first.phase, "Running");
}

// One sweep holding a NOT_FOUND pod AND a pod that changed earlier in the same sweep: the per-slot seed of the
// NOT_FOUND branch must not absorb the other pod's staged change (it did when the branch re-seeded the whole table).
static void TestSweepNotFoundDoesNotAbsorbOtherChanges() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 64);
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase); });
    for (const char* n : {"a0", "b1", "c2"}) prov.CreatePod(MakePod(n, {{PortsAnnotation, "22/tcp"}}));  // keys sort a0 < b1 < c2
    prov.UpdateAllPodStatuses();
    notified.clear();
    api->status["rp-1"].DesiredStatus = "RUNNING"; api->status["rp-1"].PortMappings["22"] = 1;  // a0: STARTING -> RUNNING (+ports)
    api->status["rp-2"].DesiredStatus = "NOT_FOUND";                                            // b1 vanishes in the same sweep
    api->status["rp-3"].DesiredStatus = "EXITED";                                               // c2 changes after the NOT_FOUND pod
    prov.UpdateAllPodStatuses();
    std::set<std::string> s(notified.begin(), notified.end());
    CHECK_EQ(notified.size(), 3u);
    CHECK(s.count("a0:Running") == 1); CHECK(s.count("b1:Failed") == 1); CHECK(s.count("c2:Succeeded") == 1);
    CHECK_EQ(prov.Info("default", "a0")->Status, "RUNNING"); CHECK(prov.Info("default", "a0")->PortsExposed);
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
    // CreatePod between two sweeps seeds ONE slot: a change staged for another pod in the next sweep still reports
    api->status["rp-1"].DesiredStatus = "TERMINATING";
    prov.CreatePod(MakePod("d3"));
    prov.UpdateAllPodStatuses();
    s = std::set<std::string>(notified.begin(), notified.end());
    CHECK(s.count("a0:Running") == 1);  // TERMINATING keeps phase Running, but it IS a status change (kubelet.go:870)
    CHECK_EQ(prov.Info("default", "a0")->Status, "TERMINATING");
}

// Status strings that do not fit the 16-byte slot: the table widens before the next sweep (32, 64, ... 256 bytes);
// beyond any slot the pod is compared on the host.  Either way the change is reported like the reference would (:870).
static void TestLongStatusStrings() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 32);
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase + ":" + p->status.container_message); });
    for (int i = 0; i < 4; ++i) prov.CreatePod(MakePod("l" + std::to_string(i)));
    prov.UpdateAllPodStatuses();
    notified.clear();
    CHECK_EQ(prov.Stride(), 16u);
    const std::string s20 = "MIGRATING_TO_NEW_HOST", s200(200, 'Q');
    api->status["rp-1"].DesiredStatus = s20;  // 21 chars: needs the 32-byte slot
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "l0:Unknown:Unknown RunPod status: " + s20);  // default: branch, :1971-1979
    CHECK_EQ(prov.Info("default", "l0")->Status, s20); CHECK_EQ(prov.HostCompares(), 1u);
    notified.clear();
    prov.UpdateAllPodStatuses();  // widened now; nothing changed
    CHECK(notified.empty()); CHECK_EQ(prov.Stride(), 32u); CHECK_EQ(prov.HostCompares(), 1u);
    api->status["rp-2"].DesiredStatus = "RUNNING";
    api->status["rp-1"].DesiredStatus = "RUNNING";
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 2u);
    notified.clear();
    api->status["rp-3"].DesiredStatus = s200;  // longer than any slot: host compare for good
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(prov.Info("default", "l2")->Status, s200);
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
    api->status["rp-3"].DesiredStatus = "EXITED";
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "l2:Succeeded:");
}

// Statuses of 30 and 62 characters widen the table to 64 and 128 bytes: the sweep's wide form.  Each widening
// seeds the whole table at the new stride right before the sweep at that stride (WidenRecords), so that sweep must
// start from a clean context, not from whatever the seed's launch left behind.  125 characters (len byte 127, the most
// a record holds) still fit 128 bytes; one more is compared on the host and the table stays at 128.
static void TestWideStatusStrings() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 600);  // 600 slots: nine 64-slot streaming units and a ragged tenth
    std::vector<std::string> notified;
    prov.NotifyPods([&](const PodPtr& p) { notified.push_back(p->name + ":" + p->status.phase + ":" + p->status.container_message); });
    for (int i = 0; i < 6; ++i) prov.CreatePod(MakePod("v" + std::to_string(i)));
    prov.UpdateAllPodStatuses();
    notified.clear();
    uint64_t host = prov.HostCompares();
    const struct { size_t len; uint32_t stride; char c; } kSteps[] = {{30, 64, 'A'}, {62, 128, 'B'}};
    for (const auto& st : kSteps) {
        const std::string s(st.len, st.c), t = std::string(st.len - 1, st.c) + "Z";
        api->status["rp-1"].DesiredStatus = s;  // v0: does not fit, compared on the host this sweep, widened before the next
        prov.UpdateAllPodStatuses();
        CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "v0:Unknown:Unknown RunPod status: " + s);
        CHECK_EQ(prov.HostCompares(), ++host);
        notified.clear();
        prov.UpdateAllPodStatuses();  // WidenRecords(stride), then the sweep at the new stride: nothing changed
        CHECK_EQ(prov.Stride(), st.stride); CHECK(notified.empty()); CHECK_EQ(prov.HostCompares(), host);
        api->status["rp-2"].DesiredStatus = t;  // v1: same length, differs in the last byte -- exactly v1, through the kernel
        prov.UpdateAllPodStatuses();
        CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "v1:Unknown:Unknown RunPod status: " + t);  // default: branch, :1971-1979
        CHECK_EQ(prov.HostCompares(), host); CHECK_EQ(prov.Info("default", "v1")->Status, t);
        notified.clear();
        prov.UpdateAllPodStatuses();
        CHECK(notified.empty());
    }
    const std::string s125(125, 'C'), s126(126, 'D');
    api->status["rp-3"].DesiredStatus = s125;  // v2: fits the 128-byte slot
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(notified[0], "v2:Unknown:Unknown RunPod status: " + s125);
    CHECK_EQ(prov.HostCompares(), host); CHECK_EQ(prov.Stride(), 128u);
    notified.clear();
    api->status["rp-3"].DesiredStatus = s126;  // longer than any slot: host compare, no widening
    prov.UpdateAllPodStatuses();
    CHECK_EQ(notified.size(), 1u); CHECK_EQ(prov.HostCompares(), host + 1);
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty()); CHECK_EQ(prov.Stride(), 128u);
    // back to a known status: Running (no ports requested, so they count as exposed)
    for (const char* id : {"rp-1", "rp-2", "rp-3"}) api->status[id].DesiredStatus = "RUNNING";
    prov.UpdateAllPodStatuses();
    std::set<std::string> s(notified.begin(), notified.end());
    CHECK_EQ(notified.size(), 3u); CHECK(s.count("v0:Running:") == 1); CHECK(s.count("v1:Running:") == 1); CHECK(s.count("v2:Running:") == 1);
    notified.clear();
    prov.UpdateAllPodStatuses();
    CHECK(notified.empty());
}

// CreatePod / DeletePod on other threads while sweeps run (the reference: pod worker + two tickers + API handlers,
// kubelet.go:374-376, 718): every status transition the fake API makes must reach notifyFunc exactly once, and device
// and host state must agree afterwards (a final quiet sweep reports nothing).
static void TestConcurrentCreateAndSweep() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    Provider prov(api, 1, 4096);
    std::mutex m;
    std::map<std::string, int> running_seen;
    prov.NotifyPods([&](const PodPtr& p) { if (p->status.phase == "Running") { std::lock_guard<std::mutex> g(m); ++running_seen[p->name]; } });
    for (int i = 0; i < 200; ++i) prov.CreatePod(MakePod("t" + std::to_string(i)));
    prov.UpdateAllPodStatuses();
    std::atomic<bool> stop{false};
    std::thread churn([&] {  // unrelated pods come and go the whole time
        int k = 0;
        while (!stop) {
            auto p = MakePod("churn" + std::to_string(k % 50));
            prov.CreatePod(p);
            if (k % 3 == 0) prov.DeletePod(prov.GetPod("default", p->name).first ? prov.GetPod("default", p->name).first : p);
            ++k;
        }
    });
    for (int round = 0; round < 20; ++round) {
        for (int i = round * 10; i < round * 10 + 10; ++i) api->SetStatus("rp-" + std::to_string(i + 1), "RUNNING");
        prov.UpdateAllPodStatuses();
    }
    stop = true;
    churn.join();
    prov.UpdateAllPodStatuses();
    int lost = 0, dup = 0;
    for (int i = 0; i < 200; ++i) {
        std::lock_guard<std::mutex> g(m);
        const int n = running_seen["t" + std::to_string(i)];
        lost += n == 0; dup += n > 1;
    }
    CHECK_EQ(lost, 0); CHECK_EQ(dup, 0);
    std::vector<std::string> late;
    prov.NotifyPods([&](const PodPtr& p) { late.push_back(p->name); });
    prov.UpdateAllPodStatuses();
    for (auto& n : late) CHECK(n.rfind("churn", 0) == 0);  // only pods the churn thread left half-way may still move
}

// self_tick: the provider drives its own sweeps like the reference's goroutines (kubelet.go:292-303, 718-729, 734-745)
static void TestSelfTick() {
    auto api = std::make_shared<FakeRunPod>();
    api->types = KatTable();
    ProviderOptions opt;
    opt.self_tick = true; opt.notify_interval_s = 0.02; opt.periodic_interval_s = 0.05; opt.pending_interval_s = 0.03;
    Provider prov(api, 1, 64, opt);
    std::mutex m;
    std::vector<std::string> notified;
    api->fail_deploy = true;
    prov.CreatePod(MakePod("late"));  // deploy fails now ...
    api->fail_deploy = false;         // ... the pending-pod ticker retries it on its own
    prov.NotifyPods([&](const PodPtr& p) { std::lock_guard<std::mutex> g(m); notified.push_back(p->name + ":" + p->status.phase); });
    bool deployed = false, running = false;
    for (int i = 0; i < 400 && !running; ++i) {
        std::this_thread::sleep_for(std::chrono::milliseconds(10));
        auto p = prov.GetPod("default", "late").first;
        if (!deployed && p && p->annotations.count(PodIDAnnotation)) { deployed = true; api->SetStatus(p->annotations.at(PodIDAnnotation), "RUNNING"); }
        std::lock_guard<std::mutex> g(m);
        for (auto& n : notified) running = running || n == "late:Running";
    }
    CHECK(deployed); CHECK(running);
    prov.StopTickers();
}

// ---- batched column ingest (no GPU) ------------------------------------------------------------------------
// Synthetic pods with the annotation shapes the reference's tests use: pod annotation, empty pod annotation with a
// Job fallback, garbage, nothing at all; the extension annotations on a minority.
static std::vector<PodPtr> SyntheticPods(size_t P, uint64_t seed) {
    static const char* kMem[] = {"2", "8", "16", "24", "40", "48", "80", "", "abc", "24GB", "99999999999", "-4"};
    static const char* kCloud[] = {"SECURE", "COMMUNITY", "community", "STANDARD", "", "secure"};
    auto job_a = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "24"}, {CloudTypeAnnotation, "COMMUNITY"}});
    auto job_b = std::make_shared<Annotations>(Annotations{{GpuMemoryAnnotation, "8"}, {VcpuAnnotation, "16"}});
    std::vector<PodPtr> pods;
    pods.reserve(P);
    uint64_t x = seed * 0x9E3779B97F4A7C15ull + 1;
    auto rnd = [&]() { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
    for (size_t i = 0; i < P; ++i) {
        Annotations a;
        const uint64_t r = rnd();
        if (r & 1) a[GpuMemoryAnnotation] = kMem[(r >> 8) % 12];
        if (r & 2) a[CloudTypeAnnotation] = kCloud[(r >> 16) % 6];
        if ((r & 0x1C) == 0x1C) a[MaxPriceAnnotation] = (r >> 24) & 1 ? "1.25" : "not-a-price";
        if ((r & 0xE0) == 0xE0) { a[VcpuAnnotation] = "32"; a[RamAnnotation] = (r >> 25) & 1 ? "128" : ""; }
        a[TemplateIdAnnotation] = "tmpl";  // annotations the path does not read are there too
        std::shared_ptr<Annotations> job = ((r >> 32) % 4 == 0) ? job_a : ((r >> 32) % 4 == 1) ? job_b : nullptr;
        pods.push_back(MakePod("p" + std::to_string(i), std::move(a), job));
    }
    return pods;
}

// PrepareRunPodParameters' annotation half spelled with the public, reference-shaped functions only (each pinned by
// the reference's own test assertions in TestColumnProducers): the yardstick for the fast row producer.
static PodColumns ColumnsByTheBook(const Pod& pod) {
    PodColumns c;
    c.cloud_type = ValidateCloudType(GetAnnotationWithFallback(pod, CloudTypeAnnotation, ""));      // runpod_client.go:1261
    c.cloud = c.cloud_type == "COMMUNITY" ? RPK_CLOUD_COMMUNITY : RPK_CLOUD_SECURE;
    const long long m = ExtractGPUMemory(GetAnnotationWithFallback(pod, GpuMemoryAnnotation, ""));  // :1277-1278
    c.req_mem_gb = m > INT32_MAX ? INT32_MAX : m < INT32_MIN ? INT32_MIN : (int32_t)m;
    auto atoi_or_zero = [](const std::string& s) -> int32_t {  // strconv.Atoi, 0 on error; saturated to the int32 column
        if (s.empty()) return 0;
        errno = 0;
        char* end = nullptr;
        const long long v = std::strtoll(s.c_str(), &end, 10);
        if (errno != 0 || *end != '\0' || std::isspace((unsigned char)s[0])) return 0;
        return v > INT32_MAX ? INT32_MAX : v < INT32_MIN ? INT32_MIN : (int32_t)v;
    };
    c.req_vcpu = atoi_or_zero(GetAnnotationWithFallback(pod, VcpuAnnotation, ""));
    c.req_ram_gb = atoi_or_zero(GetAnnotationWithFallback(pod, RamAnnotation, ""));
    c.max_price = DefaultMaxPrice;                                                                   // :48, :1281
    const std::string mp = GetAnnotationWithFallback(pod, MaxPriceAnnotation, "");
    if (!mp.empty()) {
        char* end = nullptr;
        errno = 0;
        const double d = std::strtod(mp.c_str(), &end);
        if (errno == 0 && *end == '\0' && end != mp.c_str()) c.max_price = d;
    }
    return c;
}

static void TestColumnsBatch() {
    {   // the fast row producer against the by-the-book composition, every synthetic annotation shape
        const auto pods = SyntheticPods(30000, 3);
        size_t bad = 0, community = 0, defaults = 0;
        for (const auto& p : pods) {
            const PodColumns a = PrepareColumns(*p), b = ColumnsByTheBook(*p);
            bad += !(a.req_mem_gb == b.req_mem_gb && a.req_vcpu == b.req_vcpu && a.req_ram_gb == b.req_ram_gb && a.max_price == b.max_price &&
                     a.cloud == b.cloud && a.cloud_type == b.cloud_type);
            community += a.cloud == RPK_CLOUD_COMMUNITY;
            defaults += a.req_mem_gb == 16 && a.max_price == 0.5;
        }
        CHECK_EQ(bad, 0u);
        CHECK(community > 1000 && community < 29000);  // the generator really exercises both branches
        CHECK(defaults > 1000);
    }
    for (size_t P : {(size_t)0, (size_t)1, (size_t)5000, (size_t)40000}) {
        const auto pods = SyntheticPods(P, 7 + P);
        for (int threads : {0, 1, 3, 8}) {
            PodColumnsSoA soa;
            PrepareColumnsBatch(pods, &soa, threads);
            CHECK_EQ(soa.size(), P);
            size_t bad = 0;
            for (size_t i = 0; i < P; ++i) {
                const PodColumns c = PrepareColumns(*pods[i]);
                bad += !(soa.req_mem_gb[i] == c.req_mem_gb && soa.req_vcpu[i] == c.req_vcpu && soa.req_ram_gb[i] == c.req_ram_gb &&
                         soa.max_price[i] == c.max_price && soa.cloud[i] == c.cloud);
            }
            CHECK_EQ(bad, 0u);
        }
    }
}

#include <chrono>
// host_test --bench-columns [P] : what the caller side of the grid costs on this host (annotations -> columns)
static int BenchColumns(size_t P) {
    using clk = std::chrono::steady_clock;
    const auto pods = SyntheticPods(P, 99);
    auto secs = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double>(b - a).count(); };
    PodColumnsSoA soa;
    double best1 = 1e30;
    for (int rep = 0; rep < 3; ++rep) {
        const auto t0 = clk::now();
        PrepareColumnsBatch(pods, &soa, 1);
        best1 = std::min(best1, secs(t0, clk::now()));
    }
    std::printf("{\"bench\": \"PrepareColumnsBatch\", \"pods\": %zu, \"threads\": 1, \"seconds\": %.6f, \"pods_per_s\": %.3e}\n", P, best1, P / best1);
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    for (unsigned t = 2; t <= hw; t *= 2) {
        double best = 1e30;
        for (int rep = 0; rep < 3; ++rep) {
            const auto t0 = clk::now();
            PrepareColumnsBatch(pods, &soa, (int)t);
            best = std::min(best, secs(t0, clk::now()));
        }
        std::printf("{\"bench\": \"PrepareColumnsBatch\", \"pods\": %zu, \"threads\": %u, \"seconds\": %.6f, \"pods_per_s\": %.3e}\n", P, t, best, P / best);
    }
    // the status side: one 32-byte record per tracked pod per sweep
    std::vector<uint8_t> recs(P * 32);
    static const char* kStatus[] = {"RUNNING", "STARTING", "EXITED", "TERMINATING", "TERMINATED", "NOT_FOUND"};
    double beste = 1e30;
    for (int rep = 0; rep < 3; ++rep) {
        const auto t0 = clk::now();
        for (size_t i = 0; i < P; ++i) EncodeStatusRecord(&recs[i * 32], 32, kStatus[i % 6], (i & 1) != 0);
        beste = std::min(beste, secs(t0, clk::now()));
    }
    std::printf("{\"bench\": \"EncodeStatusRecord\", \"slots\": %zu, \"threads\": 1, \"seconds\": %.6f, \"slots_per_s\": %.3e}\n", P, beste, P / beste);
    return 0;
}

int main(int argc, char** argv) {
    if (argc > 1 && std::strcmp(argv[1], "--bench-columns") == 0) return BenchColumns(argc > 2 ? (size_t)std::atoll(argv[2]) : 1000000);
    const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
    TestColumnProducers();
    TestColumnsBatch();
    TestPortsAndTranslate();
    if (gpu) {
        TestProviderDeployPath();
        TestProviderStatusSweep();
        TestSweepNotFoundDoesNotAbsorbOtherChanges();
        TestLongStatusStrings();
        TestWideStatusStrings();
        TestConcurrentCreateAndSweep();
        TestSelfTick();
    } else {
        // without a GPU the provider must refuse to start: there is no CPU fallback
        bool threw = false;
        try { Provider p(std::make_shared<FakeRunPod>(), 1, 16); } catch (const std::exception& e) { threw = std::strstr(e.what(), "no CPU fallback") != nullptr; }
        if (argc > 1 && std::strcmp(argv[1], "--cpu-no-device") == 0) CHECK(threw);
    }
    std::printf("%s: %d checks, %d failed (%s)\n", g_fail ? "FAILED" : "ok", g_checks, g_fail, gpu ? "gpu" : "cpu");
    return g_fail ? 1 : 0;
}
