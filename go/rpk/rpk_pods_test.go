package rpk

import (
	"reflect"
	"testing"
)

// processPendingPods (kubelet.go:747-814) selects by slot from the device pod table: unseeded rows hold the columns of a
// pod with no annotations, a seed overwrites only its rows, and SelectSlots equals Select over the same columns.
func TestSelectSlots(t *testing.T) {
	e, err := New(1)
	if err != nil {
		t.Skipf("no H100: %v", err)
	}
	defer e.Close()
	offers := &Offers{MemoryInGb: []int32{16, 24, 24, 48}, SecurePrice: []float64{.32, .36, 0, .40},
		CommunityPrice: []float64{.17, .22, .22, 0}, Flags: []uint8{3, 3, 2, 1}}
	if err := e.UploadOffers(offers); err != nil {
		t.Fatal(err)
	}
	if err := e.PodsReset(64); err != nil {
		t.Fatal(err)
	}
	// slot 3: 24 GB COMMUNITY, slot 9: 48 GB SECURE; every other slot keeps the defaults (16 GB SECURE)
	if err := e.PodsSeedSlots([]uint32{3, 9}, &Pods{ReqMemGb: []int32{24, 48}, Cloud: []uint8{CloudCommunity, CloudSecure}}); err != nil {
		t.Fatal(err)
	}
	slots := []uint32{9, 3, 0, 3, 63}
	got, gotTop5, err := e.SelectSlots(slots, true)
	if err != nil {
		t.Fatal(err)
	}
	cols := &Pods{ReqMemGb: []int32{48, 24, 16, 24, 16}, Cloud: []uint8{CloudSecure, CloudCommunity, CloudSecure, CloudCommunity, CloudSecure}}
	want, wantTop5, err := e.Select(cols, true)
	if err != nil {
		t.Fatal(err)
	}
	if !reflect.DeepEqual(got, want) || !reflect.DeepEqual(gotTop5, wantTop5) {
		t.Errorf("SelectSlots = %v %v, Select over the same columns = %v %v", got, gotTop5, want, wantTop5)
	}
	if err := e.PodsSeedSlots([]uint32{9, 3}, &Pods{ReqMemGb: []int32{16, 16}}); err == nil {
		t.Error("a seed that is not ascending was accepted")
	}
	if _, _, err := e.SelectSlots([]uint32{0, 64}, false); err == nil {
		t.Error("a slot outside the pod table was accepted")
	}
}
