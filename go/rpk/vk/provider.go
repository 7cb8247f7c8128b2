// Package vk is the drop-in half that keeps the virtual-kubelet surface: a Provider with the seven
// PodLifecycleHandler / PodNotifier signatures of pkg/virtual_kubelet (kubelet.go:384,421,621,654,670,699,713),
// whose two data-parallel loop bodies go through the rpk engine instead of per-pod Go loops:
//
//	processPendingPods  (kubelet.go:747-814)  one Engine.SelectSlots over ALL pending pods per tick, after
//	                                          Engine.PodsSeedSlots of the rows whose columns changed
//	updateAllPodStatuses (kubelet.go:816-974) one Engine.StatusDiffSlots over the slots fetched this tick
//
// NOT BUILT IN THIS REPOSITORY: the image has no Go toolchain and the reference's dependencies (client-go,
// virtual-kubelet v1.9.0) are not vendored (SURVEY.md 8c).  The executable twin of this file is the C++ mirror
// k8s-runpod-kubelet_b200/host/provider.cc, which the test-suite drives on the GPU; this file shows a maintainer
// where each call lands (INTEGRATION.md).  Everything network-facing stays behind RunPodAPI, as in the mirror.
package vk

import (
	"context"
	"fmt"
	"sort"
	"strings"
	"sync"
	"time"

	v1 "k8s.io/api/core/v1"

	"github.com/bsvogler/k8s-runpod-kubelet/pkg/rpk"
)

// Annotation schema, unchanged (runpod_client.go:37-52).
const (
	PodIDAnnotation     = "runpod.io/pod-id"
	CostAnnotation      = "runpod.io/cost-per-hr"
	CloudTypeAnnotation = "runpod.io/cloud-type"
	GpuMemoryAnnotation = "runpod.io/required-gpu-memory"
	PortsAnnotation     = "runpod.io/ports"
)

// InstanceInfo mirrors runpod_client.go:98-109 plus the slot of the device-resident previous-state column.
type InstanceInfo struct {
	ID             string
	CostPerHr      float64
	Status         string
	StatusMessage  string
	CreationTime   time.Time
	RequestedPorts []string
	PortsExposed   bool
	slot           uint32
}

// DetailedStatus is what GetDetailedPodStatus returns (runpod_client.go:773).
type DetailedStatus struct {
	DesiredStatus string
	PortMappings  map[string]int
}

// RunPodAPI is the out-of-scope transport (runpod_client.go:160-843).
type RunPodAPI interface {
	FetchGPUTypes() (*rpk.Offers, error)
	DeployPod(pod *v1.Pod, gpuTypeIDs []string, minRAMPerGPU int, cloudType string) (id string, costPerHr float64, err error)
	GetDetailedPodStatus(id string) (*DetailedStatus, error)
	TerminatePod(id string) error
	OwnerJobAnnotations(pod *v1.Pod) map[string]string
}

const stride = 16 // every RunPod status fits the 16-byte slot; see the C++ mirror for the widening path

// Provider implements node.PodLifecycleHandler and node.PodNotifier.
type Provider struct {
	api     RunPodAPI
	engine  *rpk.Engine
	offers  *rpk.Offers
	maxPods int

	podsMutex sync.RWMutex // kubelet.go:38-45
	pods      map[string]*v1.Pod
	podStatus map[string]*InstanceInfo
	records   []byte   // maxPods x stride: what InstanceInfo says per slot
	slotKey   []string // slot -> pod key
	freeSlots []uint32

	seedMutex sync.Mutex // the device pod table and its mirror: one deployBatch seeds and selects at a time
	seededMem []int32    // maxPods: the columns the device pod table holds per slot
	seededCld []uint8

	notifyMutex sync.RWMutex
	notifyFunc  func(*v1.Pod)
	sweepMutex  sync.Mutex // one sweep at a time (two tickers reach it: kubelet.go:292-303, 718-729)
}

// NewProvider refuses to start without the engine: there is no CPU fallback.
func NewProvider(api RunPodAPI, nGPUs, maxPods int) (*Provider, error) {
	e, err := rpk.New(nGPUs)
	if err != nil {
		return nil, fmt.Errorf("rpk engine unavailable (no CPU fallback): %w", err)
	}
	p := &Provider{api: api, engine: e, maxPods: maxPods, pods: map[string]*v1.Pod{}, podStatus: map[string]*InstanceInfo{},
		records: make([]byte, maxPods*stride), slotKey: make([]string, maxPods)}
	for s := maxPods; s > 0; s-- {
		p.freeSlots = append(p.freeSlots, uint32(s-1))
	}
	if err := e.StatusReset(maxPods); err != nil {
		return nil, err
	}
	if err := e.StatusSeed(p.records, stride); err != nil { // empty slots hold the all-zero record: they never report
		return nil, err
	}
	if err := e.PodsReset(maxPods); err != nil { // every slot: the columns of a pod with no annotations
		return nil, err
	}
	p.seededMem, p.seededCld = make([]int32, maxPods), make([]uint8, maxPods)
	for s := range p.seededMem {
		p.seededMem[s], p.seededCld[s] = 16, rpk.CloudSecure
	}
	go p.tick(30*time.Second, p.updateAllPodStatuses) // startPeriodicStatusUpdates, kubelet.go:292-303
	go p.tick(30*time.Second, p.processPendingPods)   // startPendingPodProcessor, kubelet.go:734-745
	return p, nil
}

func (p *Provider) tick(d time.Duration, f func()) {
	t := time.NewTicker(d)
	defer t.Stop()
	for range t.C {
		f()
	}
}

func key(pod *v1.Pod) string { return fmt.Sprintf("%s-%s", pod.Namespace, pod.Name) } // kubelet.go:386

// CreatePod -- kubelet.go:384-418.
func (p *Provider) CreatePod(ctx context.Context, pod *v1.Pod) error {
	k := key(pod)
	p.podsMutex.Lock()
	info, ok := p.podStatus[k]
	if !ok {
		if len(p.freeSlots) == 0 {
			p.podsMutex.Unlock()
			return fmt.Errorf("provider pod capacity exceeded")
		}
		info = &InstanceInfo{slot: p.freeSlots[len(p.freeSlots)-1]}
		p.freeSlots = p.freeSlots[:len(p.freeSlots)-1]
	}
	*info = InstanceInfo{Status: "STARTING", CreationTime: time.Now(), RequestedPorts: requestedPorts(pod), slot: info.slot}
	p.pods[k] = pod.DeepCopy()
	p.podStatus[k] = info
	p.slotKey[info.slot] = k
	rec := p.records[int(info.slot)*stride : int(info.slot+1)*stride]
	_ = rpk.EncodeStatusRecord(rec, info.Status, false, false)
	one := append([]byte(nil), rec...)
	p.podsMutex.Unlock()
	// previous state of THIS slot only: a whole-table seed would adopt other pods' pending changes as "previous"
	_ = p.engine.StatusSeedSlots([]uint32{info.slot}, one, stride)
	p.deployBatch([]string{k}) // errors are logged and swallowed: kubelet.go:406-415
	return nil
}

// UpdatePod -- kubelet.go:421-432.
func (p *Provider) UpdatePod(ctx context.Context, pod *v1.Pod) error {
	p.podsMutex.Lock()
	defer p.podsMutex.Unlock()
	p.pods[key(pod)] = pod.DeepCopy()
	return nil
}

// DeletePod -- kubelet.go:621-651.
func (p *Provider) DeletePod(ctx context.Context, pod *v1.Pod) error {
	if id := pod.Annotations[PodIDAnnotation]; id != "" {
		_ = p.api.TerminatePod(id) // failure is only logged
	}
	k := key(pod)
	p.podsMutex.Lock()
	defer p.podsMutex.Unlock()
	if info, ok := p.podStatus[k]; ok {
		for i := range p.records[int(info.slot)*stride : int(info.slot+1)*stride] {
			p.records[int(info.slot)*stride+i] = 0
		}
		p.slotKey[info.slot] = ""
		p.freeSlots = append(p.freeSlots, info.slot)
	}
	delete(p.pods, k)
	delete(p.podStatus, k)
	return nil
}

// GetPod -- kubelet.go:654-667.
func (p *Provider) GetPod(ctx context.Context, namespace, name string) (*v1.Pod, error) {
	p.podsMutex.RLock()
	defer p.podsMutex.RUnlock()
	k := fmt.Sprintf("%s-%s", namespace, name)
	if pod, ok := p.pods[k]; ok {
		return pod, nil
	}
	return nil, fmt.Errorf("pod %s not found", k)
}

// GetPodStatus -- kubelet.go:670-696.
func (p *Provider) GetPodStatus(ctx context.Context, namespace, name string) (*v1.PodStatus, error) {
	p.podsMutex.RLock()
	defer p.podsMutex.RUnlock()
	k := fmt.Sprintf("%s-%s", namespace, name)
	pod, ok := p.pods[k]
	if !ok {
		return nil, fmt.Errorf("pod status not found for %s", k)
	}
	return &pod.Status, nil
}

// GetPods -- kubelet.go:699-710 (returns the internal pointers, as the reference does).
func (p *Provider) GetPods(ctx context.Context) ([]*v1.Pod, error) {
	p.podsMutex.RLock()
	defer p.podsMutex.RUnlock()
	out := make([]*v1.Pod, 0, len(p.pods))
	for _, pod := range p.pods {
		out = append(out, pod)
	}
	return out, nil
}

// NotifyPods -- kubelet.go:713-731: install the callback, return immediately, sweep every 10 s.
func (p *Provider) NotifyPods(ctx context.Context, notifyFunc func(*v1.Pod)) {
	p.notifyMutex.Lock()
	p.notifyFunc = notifyFunc
	p.notifyMutex.Unlock()
	go func() {
		t := time.NewTicker(10 * time.Second)
		defer t.Stop()
		for {
			select {
			case <-ctx.Done():
				return
			case <-t.C:
				p.updateAllPodStatuses()
			}
		}
	}()
}

// processPendingPods -- kubelet.go:747-814, batched: every Pending pod without a RunPod id goes into ONE select.
func (p *Provider) processPendingPods() {
	var keys []string
	p.podsMutex.RLock()
	for k, pod := range p.pods {
		if pod.Status.Phase == v1.PodPending && pod.Annotations[PodIDAnnotation] == "" {
			keys = append(keys, k)
		}
	}
	p.podsMutex.RUnlock()
	if len(keys) > 0 {
		p.deployBatch(keys)
	}
}

// seedAndSelect seeds the pod-table rows whose columns differ from what the slot holds on the device (a changed pod or
// owner Job, or a slot reused by another pod), in ascending slot order, then selects the batch by slot.  seedMutex held.
func (p *Provider) seedAndSelect(slots []uint32, cols *rpk.Pods) ([]int32, error) {
	idx := make([]int, 0, len(slots))
	for i, s := range slots {
		if cols.ReqMemGb[i] != p.seededMem[s] || cols.Cloud[i] != p.seededCld[s] {
			idx = append(idx, i)
		}
	}
	if len(idx) > 0 {
		sort.Slice(idx, func(a, b int) bool { return slots[idx[a]] < slots[idx[b]] })
		seed, seedSlots := &rpk.Pods{}, make([]uint32, 0, len(idx))
		for _, i := range idx {
			seedSlots = append(seedSlots, slots[i])
			seed.ReqMemGb = append(seed.ReqMemGb, cols.ReqMemGb[i])
			seed.Cloud = append(seed.Cloud, cols.Cloud[i])
		}
		if err := p.engine.PodsSeedSlots(seedSlots, seed); err != nil {
			return nil, err
		}
		for k, s := range seedSlots {
			p.seededMem[s], p.seededCld[s] = seed.ReqMemGb[k], seed.Cloud[k]
		}
	}
	_, top5, err := p.engine.SelectSlots(slots, true)
	return top5, err
}

func (p *Provider) deployBatch(keys []string) {
	cols := &rpk.Pods{}
	var pods []*v1.Pod
	var slots []uint32
	p.podsMutex.RLock()
	for _, k := range keys {
		pod, ok := p.pods[k]
		info, tracked := p.podStatus[k]
		if ok && tracked {
			// derived on every retry, owner Job included, as the reference does (runpod_client.go:1250-1281)
			job := p.api.OwnerJobAnnotations(pod)
			cols.ReqMemGb = append(cols.ReqMemGb, rpk.ReqMemColumn(rpk.AnnotationWithFallback(pod.Annotations, job, GpuMemoryAnnotation, "")))
			cols.Cloud = append(cols.Cloud, rpk.CloudColumn(rpk.AnnotationWithFallback(pod.Annotations, job, CloudTypeAnnotation, "")))
			pods = append(pods, pod)
			slots = append(slots, info.slot)
		}
	}
	p.podsMutex.RUnlock()
	offers, err := p.api.FetchGPUTypes() // ONE fetch per tick (the reference: one per pod, runpod_client.go:447-455)
	if err != nil {
		return
	}
	p.seedMutex.Lock()
	if p.offers == nil || !sameTable(p.offers, offers) {
		if err := p.engine.UploadOffers(offers); err != nil {
			p.seedMutex.Unlock()
			return
		}
		p.offers = offers
	}
	top5, err := p.seedAndSelect(slots, cols)
	p.seedMutex.Unlock()
	if err != nil {
		return
	}
	for i, pod := range pods {
		var ids []string // params["gpuTypeIds"], runpod_client.go:1339
		for _, g := range top5[i*rpk.TopK : (i+1)*rpk.TopK] {
			if g >= 0 {
				ids = append(ids, p.offers.IDs[g])
			}
		}
		cloud := "SECURE"
		if cols.Cloud[i] == rpk.CloudCommunity {
			cloud = "COMMUNITY"
		}
		id, cost, err := p.api.DeployPod(pod, ids, int(cols.ReqMemGb[i]), cloud)
		if err != nil {
			continue // retried by the next tick
		}
		p.podsMutex.Lock() // updatePodWithRunPodInfo, kubelet.go:505-562
		if cur, ok := p.pods[key(pod)]; ok {
			np := cur.DeepCopy()
			if np.Annotations == nil {
				np.Annotations = map[string]string{}
			}
			np.Annotations[PodIDAnnotation] = id
			np.Annotations[CostAnnotation] = fmt.Sprintf("%f", cost)
			p.pods[key(pod)] = np
			p.podStatus[key(pod)].ID, p.podStatus[key(pod)].CostPerHr = id, cost
		}
		p.podsMutex.Unlock()
	}
}

// updateAllPodStatuses -- kubelet.go:816-974, batched; see the C++ mirror for the concurrency argument.
func (p *Provider) updateAllPodStatuses() {
	p.sweepMutex.Lock()
	defer p.sweepMutex.Unlock()
	type fresh struct {
		key, status string
		ports       bool
		rec         []byte
	}
	p.podsMutex.RLock()
	type target struct {
		key  string
		pod  *v1.Pod
		info InstanceInfo
	}
	var targets []target
	for k, pod := range p.pods {
		if info, ok := p.podStatus[k]; ok {
			targets = append(targets, target{k, pod, *info})
		}
	}
	p.podsMutex.RUnlock()
	bySlot := map[uint32]fresh{}
	for _, t := range targets {
		if t.pod.Status.Phase == v1.PodSucceeded || t.pod.Status.Phase == v1.PodFailed { // :836
			continue
		}
		id := t.pod.Annotations[PodIDAnnotation]
		if id == "" { // :841-844
			continue
		}
		ds, err := p.api.GetDetailedPodStatus(id)
		if err != nil || ds.DesiredStatus == "NOT_FOUND" { // :848-864 (handleMissingRunPodInstance stays the reference's code)
			continue
		}
		ports := checkPortsExposed(ds.PortMappings, t.info.RequestedPorts) // :867
		low := strings.ToLower(t.info.StatusMessage)
		flag := strings.Contains(low, "error") || strings.Contains(low, "fail")
		rec := make([]byte, stride)
		if rpk.EncodeStatusRecord(rec, ds.DesiredStatus, ports, flag) == nil {
			bySlot[t.info.slot] = fresh{t.key, ds.DesiredStatus, ports, rec}
		}
	}
	slots := make([]uint32, 0, len(bySlot)) // the fetched slots, ascending, and their records packed in that order
	for s := range bySlot {
		slots = append(slots, s)
	}
	sort.Slice(slots, func(i, j int) bool { return slots[i] < slots[j] })
	recs := make([]byte, 0, len(slots)*stride)
	for _, s := range slots {
		recs = append(recs, bySlot[s].rec...)
	}
	changed, codes, err := p.engine.StatusDiffSlots(slots, recs, stride) // :870-873 for the fetched slots + the decision per changed slot
	if err != nil {
		return
	}
	var reseed []uint32
	for i, slot := range changed {
		f, ok := bySlot[slot]
		p.podsMutex.Lock()
		info, tracked := p.podStatus[f.key]
		if !ok || !tracked || info.slot != slot {
			p.podsMutex.Unlock()
			reseed = append(reseed, slot) // reported but not applied: device state must follow records, not the fetched one
			continue
		}
		info.Status, info.PortsExposed = f.status, f.ports // :875-880
		copy(p.records[int(slot)*stride:int(slot+1)*stride], f.rec)
		np := p.pods[f.key].DeepCopy()
		np.Status = *podStatusFromCode(codes[i], f.status, info.StatusMessage) // translateRunPodStatus, :883
		p.pods[f.key] = np
		p.podsMutex.Unlock()
		p.notifyMutex.RLock()
		nf := p.notifyFunc
		p.notifyMutex.RUnlock()
		if nf != nil {
			nf(np) // :936-954
		}
	}
	if len(reseed) > 0 {
		p.podsMutex.RLock()
		recs := make([]byte, 0, len(reseed)*stride)
		for _, s := range reseed {
			recs = append(recs, p.records[int(s)*stride:int(s+1)*stride]...)
		}
		p.podsMutex.RUnlock()
		_ = p.engine.StatusSeedSlots(reseed, recs, stride)
	}
}

// podStatusFromCode rebuilds translateRunPodStatus's v1.PodStatus (kubelet.go:1848-2024) from the kernel's code.
func podStatusFromCode(c rpk.StatusCode, status, message string) *v1.PodStatus {
	phases := [...]v1.PodPhase{v1.PodUnknown, v1.PodPending, v1.PodRunning, v1.PodSucceeded, v1.PodFailed, v1.PodUnknown, v1.PodUnknown, v1.PodUnknown}
	cs := v1.ContainerStatus{Name: "runpod-container", Image: "runpod-image", ContainerID: "runpod://", Ready: c.Ready()}
	started := c.Started()
	cs.Started = &started
	text := message
	switch c.Message() {
	case 1:
		text = "Container reported as running but ports not yet exposed" // :1885
	case 2:
		text = "Pod was deleted from RunPod API" // :1963
	case 3:
		text = fmt.Sprintf("Unknown RunPod status: %s", status) // :1975
	}
	switch c.State() {
	case 1:
		cs.State.Running = &v1.ContainerStateRunning{}
	case 2:
		cs.State.Terminated = &v1.ContainerStateTerminated{ExitCode: c.ExitCode(), Reason: rpk.Reasons[c.Reason()], Message: text}
	default:
		cs.State.Waiting = &v1.ContainerStateWaiting{Reason: rpk.Reasons[c.Reason()], Message: text}
	}
	ready := v1.ConditionFalse
	if c.Ready() {
		ready = v1.ConditionTrue // :1982-1985
	}
	return &v1.PodStatus{Phase: phases[c.Phase()], Message: message, ContainerStatuses: []v1.ContainerStatus{cs},
		Conditions: []v1.PodCondition{{Type: v1.PodScheduled, Status: v1.ConditionTrue}, {Type: v1.PodInitialized, Status: v1.ConditionTrue},
			{Type: v1.PodReady, Status: ready}, {Type: v1.ContainersReady, Status: ready}}}
}

// checkPortsExposed -- kubelet.go:566-605 (host-side string-map work; stays on the host).
func checkPortsExposed(mappings map[string]int, requested []string) bool {
	for _, rp := range requested {
		found := false
		for port := range mappings {
			if rp == port+"/tcp" || rp == port+"/http" {
				found = true
				break
			}
		}
		if !found && !strings.HasSuffix(rp, "/http") {
			return false
		}
	}
	return true
}

func requestedPorts(pod *v1.Pod) []string { // runpod_client.go:1381-1393, annotation half
	if v := pod.Annotations[PortsAnnotation]; v != "" {
		parts := strings.Split(v, ",")
		for i := range parts {
			parts[i] = strings.TrimSpace(parts[i])
		}
		return parts
	}
	return nil
}

func sameTable(a, b *rpk.Offers) bool {
	if len(a.IDs) != len(b.IDs) {
		return false
	}
	for i := range a.IDs {
		if a.IDs[i] != b.IDs[i] || a.MemoryInGb[i] != b.MemoryInGb[i] || a.SecurePrice[i] != b.SecurePrice[i] ||
			a.CommunityPrice[i] != b.CommunityPrice[i] || a.Flags[i] != b.Flags[i] {
			return false
		}
	}
	return true
}
