package rpk

import (
	"reflect"
	"testing"
)

// updateAllPodStatuses compares only the pods it fetched this cycle (kubelet.go:836-864): a slot-list diff reports
// the listed slots whose (status, ports) pair changed and leaves every other slot's previous state alone.
func TestStatusDiffSlots(t *testing.T) {
	e, err := New(1)
	if err != nil {
		t.Skipf("no H100: %v", err)
	}
	defer e.Close()
	const stride = 16
	recs := make([]byte, 4*stride)
	for i := 0; i < 4; i++ {
		if err := EncodeStatusRecord(recs[i*stride:(i+1)*stride], "STARTING", false, false); err != nil {
			t.Fatal(err)
		}
	}
	if err := e.StatusSeed(recs, stride); err != nil {
		t.Fatal(err)
	}
	// slot 1 is not fetched this cycle although its pod moved: it must not be compared
	fetched := make([]byte, 2*stride)
	_ = EncodeStatusRecord(fetched[0:stride], "RUNNING", true, false)         // slot 0 changed
	_ = EncodeStatusRecord(fetched[stride:2*stride], "STARTING", false, false) // slot 3 unchanged
	got, codes, err := e.StatusDiffSlots([]uint32{0, 3}, fetched, stride)
	if err != nil {
		t.Fatal(err)
	}
	if want := []uint32{0}; !reflect.DeepEqual(got, want) || len(codes) != 1 || codes[0].Phase() != 2 {
		t.Errorf("changed = %v codes %v, want [0] with phase Running", got, codes)
	}
	if _, _, err := e.StatusDiffSlots([]uint32{3, 0}, fetched, stride); err == nil {
		t.Error("a list that is not ascending was accepted")
	}
	// the whole table still holds slot 0's new state and everything else as seeded
	_ = EncodeStatusRecord(recs[0:stride], "RUNNING", true, false)
	if got, err := e.StatusDiff(recs, stride); err != nil || len(got) != 0 {
		t.Errorf("whole-table sweep reported %v (err %v)", got, err)
	}
}
