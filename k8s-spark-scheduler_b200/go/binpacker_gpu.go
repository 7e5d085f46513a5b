//go:build cgo

// Package binpackergpu is the cgo shim a maintainer of palantir/k8s-spark-scheduler adds to route the
// placement hot path through libgangpack.so (include/gangpack.h).
//
// NOT COMPILED OR TESTED HERE: this environment has no Go toolchain.  The same marshalling, written in
// C++ and exercised on an H100, is k8s-spark-scheduler_b200/host/gangpack_host.hpp; this file is kept
// deliberately thin so that the two can be compared line by line.  See INTEGRATION.md.
//
// Build: CGO_ENABLED=1 (the reference builds with CGO_ENABLED=0, godel/config/dist-plugin.yml:7,26),
//
//	CGO_CFLAGS=-I<repo>/include  CGO_LDFLAGS="-L<repo>/k8s-spark-scheduler_b200 -lgangpack"
package binpackergpu

/*
#include <stdlib.h>
#include "gangpack.h"
*/
import "C"

import (
	"context"
	"fmt"
	"math"
	"runtime"
	"sort"
	"strconv"
	"sync"
	"unsafe"

	"github.com/palantir/k8s-spark-scheduler-lib/pkg/binpack"
	"github.com/palantir/k8s-spark-scheduler-lib/pkg/resources"
	"github.com/palantir/k8s-spark-scheduler/internal/common"
	v1 "k8s.io/api/core/v1"
	"k8s.io/apimachinery/pkg/api/resource"
	"k8s.io/apimachinery/pkg/labels"
	"k8s.io/apimachinery/pkg/selection"
	clientcache "k8s.io/client-go/tools/cache"
)

// Names under which the GPU packers are registered next to the reference's own entries in
// internal/binpacker.binpackFunctions (internal/binpacker/binpack.go:43-49).  Registering them under
// the existing names "tightly-pack" / "distribute-evenly" instead makes cmd/server.go:145 pick them
// with an unchanged install.yml.
const (
	TightlyPackGPU      = "tightly-pack-gpu"
	DistributeEvenlyGPU = "distribute-evenly-gpu"
)

// device owns one gp_ctx; Predicate is serial (internal/extender/resource.go:194-205) but the
// unschedulable-pod marker calls BinpackFunc from its own goroutine (cmd/server.go:230), hence the mutex.
type device struct {
	mu  sync.Mutex
	ctx *C.gp_ctx
}

var (
	dev     *device
	devOnce sync.Once
	devErr  error
)

func getDevice() (*device, error) {
	devOnce.Do(func() {
		var ctx *C.gp_ctx
		if st := C.gp_create(&ctx, nil); st != C.GP_OK {
			devErr = fmt.Errorf("gp_create: %s", C.GoString(C.gp_last_error(nil)))
			return
		}
		dev = &device{ctx: ctx}
	})
	return dev, devErr
}

// milli converts a Quantity to the exact-int64 model; ok=false routes the call to the Go packer
// (Quantity falls back to inf.Dec beyond int64 / for sub-milli scales, quantity.go:556-591).
func milli(q resource.Quantity) (int64, bool) {
	if q.Cmp(*resource.NewMilliQuantity(q.MilliValue(), q.Format)) != 0 {
		return 0, false
	}
	return q.MilliValue(), true
}
func whole(q resource.Quantity) (int64, bool) {
	v, ok := q.AsInt64()
	return v, ok
}

func toTriple(r *resources.Resources) (cpu, mem, gpu int64, ok bool) {
	var a, b, c bool
	cpu, a = milli(r.CPU)
	mem, b = whole(r.Memory)
	gpu, c = whole(r.NvidiaGPU)
	return cpu, mem, gpu, a && b && c
}

// snapshot marshals the metadata map and the two priority orders into SoA buffers.  Names that are
// not in the metadata are dropped: they can host neither a driver (binpack.go:68-69) nor an executor
// (pack_tightly.go:51-52).
type snapshot struct {
	names            []string
	cpu, mem, gpu    []int64
	execIdx, drvIdx  []int32
}

func marshal(md resources.NodeGroupSchedulingMetadata, driverOrder, executorOrder []string) (*snapshot, bool) {
	s := &snapshot{}
	index := make(map[string]int32, len(md))
	intern := func(n string) (int32, bool, bool) {
		if i, ok := index[n]; ok {
			return i, true, true
		}
		m, ok := md[n]
		if !ok {
			return -1, false, true
		}
		c, mm, g, exact := toTriple(m.AvailableResources)
		if !exact {
			return -1, false, false
		}
		i := int32(len(s.names))
		index[n] = i
		s.names = append(s.names, n)
		s.cpu, s.mem, s.gpu = append(s.cpu, c), append(s.mem, mm), append(s.gpu, g)
		return i, true, true
	}
	for _, n := range executorOrder {
		i, present, exact := intern(n)
		if !exact {
			return nil, false
		}
		if present {
			s.execIdx = append(s.execIdx, i)
		}
	}
	for _, n := range driverOrder {
		i, present, exact := intern(n)
		if !exact {
			return nil, false
		}
		if present {
			s.drvIdx = append(s.drvIdx, i)
		}
	}
	return s, true
}

func ptr64(v []int64) *C.int64_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.int64_t)(unsafe.Pointer(&v[0]))
}
func ptr32(v []int32) *C.int32_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&v[0]))
}

func (d *device) setSnapshot(s *snapshot) error {
	eoff := []int32{0, int32(len(s.execIdx))}
	doff := []int32{0, int32(len(s.drvIdx))}
	var pin runtime.Pinner // Go >= 1.21: the struct holds Go pointers for the duration of the call
	defer pin.Unpin()
	for _, p := range []any{ptrOrNil(s.cpu), ptrOrNil(s.mem), ptrOrNil(s.gpu), ptrOrNil32(s.execIdx), ptrOrNil32(s.drvIdx), &eoff[0], &doff[0]} {
		if p != nil {
			pin.Pin(p)
		}
	}
	n := C.gp_nodes{
		n_nodes: C.int32_t(len(s.names)), avail_cpu_milli: ptr64(s.cpu), avail_mem_bytes: ptr64(s.mem), avail_gpu: ptr64(s.gpu),
		n_groups: 1, exec_off: ptr32(eoff), exec_order: ptr32(s.execIdx), drv_off: ptr32(doff), drv_order: ptr32(s.drvIdx),
	}
	if st := C.gp_set_snapshot(d.ctx, &n); st != C.GP_OK {
		return fmt.Errorf("gp_set_snapshot: %s", C.GoString(C.gp_last_error(d.ctx)))
	}
	return nil
}

func ptrOrNil(v []int64) any {
	if len(v) == 0 {
		return nil
	}
	return &v[0]
}
func ptrOrNil32(v []int32) any {
	if len(v) == 0 {
		return nil
	}
	return &v[0]
}
func ptrOrNil8(v []uint8) any {
	if len(v) == 0 {
		return nil
	}
	return &v[0]
}
func ptr8(v []uint8) *C.uint8_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&v[0]))
}

// gpuPacker returns a binpack.SparkBinPackFunction (LIB/binpack/binpack.go:43-48) backed by the device;
// any failure (no device, CUDA error, unrepresentable quantity) runs `fallback`, the original Go packer,
// so Predicate never fails because of the accelerator.
func gpuPacker(algo C.gp_algo, fallback binpack.SparkBinPackFunction) binpack.SparkBinPackFunction {
	return func(ctx context.Context, driverResources, executorResources *resources.Resources, executorCount int,
		driverNodePriorityOrder, executorNodePriorityOrder []string,
		nodesSchedulingMetadata resources.NodeGroupSchedulingMetadata) *binpack.PackingResult {
		goPath := func() *binpack.PackingResult {
			return fallback(ctx, driverResources, executorResources, executorCount, driverNodePriorityOrder,
				executorNodePriorityOrder, nodesSchedulingMetadata)
		}
		d, err := getDevice()
		if err != nil {
			return goPath()
		}
		dc, dm, dg, ok1 := toTriple(driverResources)
		ec, em, eg, ok2 := toTriple(executorResources)
		s, ok3 := marshal(nodesSchedulingMetadata, driverNodePriorityOrder, executorNodePriorityOrder)
		if !ok1 || !ok2 || !ok3 || executorCount < 0 {
			return goPath()
		}
		runtime.LockOSThread()
		defer runtime.UnlockOSThread()
		d.mu.Lock()
		defer d.mu.Unlock()
		if err := d.setSnapshot(s); err != nil {
			return goPath()
		}
		nodes := make([]int32, max(executorCount, 1))
		var has, driver C.int32_t
		st := C.gp_pack_one(d.ctx, algo, C.int64_t(dc), C.int64_t(dm), C.int64_t(dg), C.int64_t(ec), C.int64_t(em), C.int64_t(eg),
			C.int32_t(executorCount), &has, &driver, ptr32(nodes))
		if st != C.GP_OK {
			return goPath()
		}
		if has == 0 {
			return binpack.EmptyPackingResult()
		}
		res := &binpack.PackingResult{DriverNode: s.names[driver], HasCapacity: true,
			ExecutorNodes: make([]string, executorCount)}
		for i := 0; i < executorCount; i++ {
			res.ExecutorNodes[i] = s.names[nodes[i]]
		}
		// PackingEfficiencies (metrics/debug log only for these two packers, EXT/resource.go:329-352) are
		// computed on the host from the result when a caller asks for them:
		res.PackingEfficiencies = efficienciesFor(nodesSchedulingMetadata, driverResources, executorResources, res,
			algo != C.GP_MINIMAL_FRAGMENTATION)
		return res
	}
}

// efficienciesFor rebuilds the reserved map of SparkBinPack (binpack.go:72-77) from the placement and
// calls the reference's own ComputePackingEfficiencies.  tightlyPackExecutors / distributeExecutorsEvenly add every
// executor to that map; minimalFragmentation never touches it (withExecutors=false), which is what the reference's
// chooseBestResult then sees -- kept as is.
func efficienciesFor(md resources.NodeGroupSchedulingMetadata, drv, exe *resources.Resources, r *binpack.PackingResult,
	withExecutors bool) map[string]*binpack.PackingEfficiency {
	reserved := resources.NodeGroupResources{r.DriverNode: drv.Copy()}
	if withExecutors {
		for _, n := range r.ExecutorNodes {
			if reserved[n] == nil {
				reserved[n] = resources.Zero()
			}
			reserved[n].Add(exe)
		}
	}
	return binpack.ComputePackingEfficiencies(md, reserved)
}

// AvgPackingEfficiencyForResult is computeAvgPackingEfficiencyForResult (EXT/resource.go:372-381), the metric the
// Predicate reports at :352, over EVERY node of nodesSchedulingMetadata -- the metadata the packer saw -- with `reserved`
// rebuilt from the placement (minimalFragmentation: the driver only).  It marshals the whole node table (availability and
// SchedulableResources, every node as an executor candidate so the snapshot covers them all), uploads it and makes ONE
// gp_packing_efficiency call; it never relies on a snapshot an earlier call left on the context, whose node table may be
// another one (the packers here upload only the nodes of their priority orders).  The sums are rounded once from their
// exact value: the Go loop sums in map order, so the two agree within the recursive-summation bound (bit for bit when
// every partial sum is exact).  A shim that keeps a gp_prepare_cluster / gp_prepare_cluster_zones snapshot resident calls
// gp_packing_efficiency on it directly instead (INTEGRATION.md, the Predicate recipe's step 4).
// ok=false (no device, a name outside the metadata, an inexact quantity, a device error): the caller runs the Go
// computeAvgPackingEfficiencyForResult on the PackingEfficiencies the Go packer returns.
func AvgPackingEfficiencyForResult(nodesSchedulingMetadata resources.NodeGroupSchedulingMetadata,
	driverResources, executorResources *resources.Resources, result *binpack.PackingResult,
	minimalFragmentation bool) (binpack.AvgPackingEfficiency, bool) {
	if result == nil || !result.HasCapacity {
		return binpack.WorstAvgPackingEfficiency(), true
	}
	d, err := getDevice()
	if err != nil {
		return binpack.AvgPackingEfficiency{}, false
	}
	dc, dm, dg, ok1 := toTriple(driverResources)
	ec, em, eg, ok2 := toTriple(executorResources)
	if !ok1 || !ok2 {
		return binpack.AvgPackingEfficiency{}, false
	}
	all := make([]string, 0, len(nodesSchedulingMetadata))
	for n := range nodesSchedulingMetadata {
		all = append(all, n)
	}
	s, ok := marshal(nodesSchedulingMetadata, nil, all)
	if !ok {
		return binpack.AvgPackingEfficiency{}, false
	}
	index := make(map[string]int32, len(s.names))
	sc, sm, sg := make([]int64, len(s.names)+1), make([]int64, len(s.names)+1), make([]int64, len(s.names)+1)
	for i, n := range s.names {
		index[n] = int32(i)
		c, m, g, exact := toTriple(nodesSchedulingMetadata[n].SchedulableResources)
		if !exact {
			return binpack.AvgPackingEfficiency{}, false
		}
		sc[i], sm[i], sg[i] = c, m, g
	}
	driver, ok := index[result.DriverNode]
	if !ok {
		return binpack.AvgPackingEfficiency{}, false
	}
	execs := make([]int32, max(len(result.ExecutorNodes), 1))
	for i, n := range result.ExecutorNodes {
		v, ok := index[n]
		if !ok {
			return binpack.AvgPackingEfficiency{}, false
		}
		execs[i] = v
	}
	drv := []int64{dc, dm, dg}
	exe := []int64{ec, em, eg}
	count := []int32{int32(len(result.ExecutorNodes))}
	off := []int64{0, int64(len(result.ExecutorNodes))}
	drvNode := []int32{driver}
	avg := make([]float64, 4)
	algo := C.gp_algo(C.GP_TIGHTLY_PACK)
	if minimalFragmentation {
		algo = C.GP_MINIMAL_FRAGMENTATION
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	if err := d.setSnapshot(s); err != nil {
		return binpack.AvgPackingEfficiency{}, false
	}
	if st := C.gp_set_schedulable(d.ctx, ptr64(sc), ptr64(sm), ptr64(sg)); st != C.GP_OK {
		return binpack.AvgPackingEfficiency{}, false
	}
	// gp_apps / gp_results hold Go pointers: every slice base is pinned for the duration of the call
	// (cgocheck: "Go pointer to unpinned Go pointer"), exactly as setSnapshot does for the node table.
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{&drv[0], &exe[0], &count[0], &off[0], &drvNode[0], &execs[0]} {
		pin.Pin(p)
	}
	a := C.gp_apps{n_apps: 1, drv_cpu_milli: ptr64(drv[0:1]), drv_mem_bytes: ptr64(drv[1:2]), drv_gpu: ptr64(drv[2:3]),
		exe_cpu_milli: ptr64(exe[0:1]), exe_mem_bytes: ptr64(exe[1:2]), exe_gpu: ptr64(exe[2:3]), exe_count: ptr32(count),
		exec_out_off: ptr64(off)}
	placed := C.gp_results{driver_node: ptr32(drvNode), executor_nodes: ptr32(execs), executor_nodes_cap: C.int64_t(len(execs))}
	if C.gp_packing_efficiency(d.ctx, &a, algo, &placed, C.GP_MODE_INDEPENDENT, (*C.double)(unsafe.Pointer(&avg[0]))) != C.GP_OK {
		return binpack.AvgPackingEfficiency{}, false
	}
	return binpack.AvgPackingEfficiency{CPU: avg[0], Memory: avg[1], GPU: avg[2], Max: avg[3]}, true
}

// TightlyPack / DistributeEvenly / MinimalFragmentation are drop-in values for binpack.TightlyPack /
// binpack.DistributeEvenly / binpack.MinimalFragmentation.
var (
	TightlyPack          = gpuPacker(C.GP_TIGHTLY_PACK, binpack.TightlyPack)
	DistributeEvenly     = gpuPacker(C.GP_DISTRIBUTE_EVENLY, binpack.DistributeEvenly)
	MinimalFragmentation = gpuPacker(C.GP_MINIMAL_FRAGMENTATION, binpack.MinimalFragmentation)
)

// singleAZ is getSingleAZSparkBinFunction + chooseBestResult (LIB/binpack/single_az.go:23-97) over a device packer
// (both are unexported in the lib, hence restated here with its exported efficiency helpers).  The C++ mirror packs all
// zones in ONE device batch (zone = instance group, host/gangpack_host.hpp SingleAZPackImpl); this thin version calls
// the per-zone packer once per zone.
func singleAZ(perZone binpack.SparkBinPackFunction) binpack.SparkBinPackFunction {
	return func(ctx context.Context, driverResources, executorResources *resources.Resources, executorCount int,
		driverNodePriorityOrder, executorNodePriorityOrder []string,
		md resources.NodeGroupSchedulingMetadata) *binpack.PackingResult {
		group := func(names []string) ([]string, map[string][]string) { // groupNodesByZone, :57-73
			order, byZone := []string{}, map[string][]string{}
			for _, n := range names {
				m, ok := md[n]
				if !ok {
					continue
				}
				if _, seen := byZone[m.ZoneLabel]; !seen {
					order = append(order, m.ZoneLabel)
				}
				byZone[m.ZoneLabel] = append(byZone[m.ZoneLabel], n)
			}
			return order, byZone
		}
		zones, dz := group(driverNodePriorityOrder)
		_, ez := group(executorNodePriorityOrder)
		best, bestAvg := binpack.EmptyPackingResult(), binpack.WorstAvgPackingEfficiency() // :79-80
		for _, z := range zones {
			eo, ok := ez[z]
			if !ok {
				continue // :38-41
			}
			r := perZone(ctx, driverResources, executorResources, executorCount, dz[z], eo, md)
			if !r.HasCapacity {
				continue // :44-46
			}
			effs := make([]*binpack.PackingEfficiency, 0, 1+len(r.ExecutorNodes)) // :83-89
			for _, n := range append([]string{r.DriverNode}, r.ExecutorNodes...) {
				effs = append(effs, r.PackingEfficiencies[n])
			}
			if avg := binpack.ComputeAvgPackingEfficiency(md, effs); bestAvg.LessThan(avg) { // :90-94
				best, bestAvg = r, avg
			}
		}
		return best
	}
}

// Drop-in values for binpack.SingleAZTightlyPack / binpack.SingleAZMinimalFragmentation / binpack.AzAwareTightlyPack.
var (
	SingleAZTightlyPack          = singleAZ(TightlyPack)
	SingleAZMinimalFragmentation = singleAZ(MinimalFragmentation)
	AzAwareTightlyPack           = binpack.SparkBinPackFunction(func(ctx context.Context, d, e *resources.Resources, k int,
		dord, eord []string, md resources.NodeGroupSchedulingMetadata) *binpack.PackingResult {
		if r, ok := azAwareTightlyPackDevice(d, e, k, dord, eord, md); ok {
			return r
		}
		return binpack.AzAwareTightlyPack(ctx, d, e, k, dord, eord, md)
	})
)

// azAwareTightlyPackDevice is AzAwareTightlyPack (LIB/binpack/az_aware_pack_tightly.go:27-38) for one application as
// ONE gp_pack_batch_az_aware call on the az-aware layout: the zone packs, the zone choice and, when no zone wins, the
// fallback over the undivided orders all run on the device.  ok=false (no device, a quantity that is not an exact int64,
// a device error): the caller runs the Go packer.
func azAwareTightlyPackDevice(driverResources, executorResources *resources.Resources, executorCount int,
	driverNodePriorityOrder, executorNodePriorityOrder []string,
	md resources.NodeGroupSchedulingMetadata) (*binpack.PackingResult, bool) {
	d, err := getDevice()
	if err != nil {
		return nil, false
	}
	dc, dm, dg, ok1 := toTriple(driverResources)
	ec, em, eg, ok2 := toTriple(executorResources)
	l, ok3 := azAwareLayout(driverNodePriorityOrder, executorNodePriorityOrder, md)
	if !ok1 || !ok2 || !ok3 || executorCount < 0 {
		return nil, false
	}
	cnt := []int32{int32(executorCount)}
	zone, driver := []int32{-1}, []int32{-1}
	exec := make([]int32, max(executorCount, 1))
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	l.pin(&pin)
	for _, p := range []any{&dc, &dm, &dg, &ec, &em, &eg, ptrOrNil32(cnt), ptrOrNil32(zone), ptrOrNil32(driver), ptrOrNil32(exec)} {
		pin.Pin(p)
	}
	if !l.upload(d) {
		return nil, false
	}
	ga := C.gp_apps{n_apps: 1, drv_cpu_milli: (*C.int64_t)(unsafe.Pointer(&dc)), drv_mem_bytes: (*C.int64_t)(unsafe.Pointer(&dm)),
		drv_gpu: (*C.int64_t)(unsafe.Pointer(&dg)), exe_cpu_milli: (*C.int64_t)(unsafe.Pointer(&ec)),
		exe_mem_bytes: (*C.int64_t)(unsafe.Pointer(&em)), exe_gpu: (*C.int64_t)(unsafe.Pointer(&eg)), exe_count: ptr32(cnt)}
	orders := l.orders()
	gz := C.gp_zone_results{zone: ptr32(zone), driver_node: ptr32(driver), executor_nodes: ptr32(exec), executor_nodes_cap: C.int64_t(len(exec))}
	if st := C.gp_pack_batch_az_aware(d.ctx, &ga, &orders, &gz); st != C.GP_OK {
		return nil, false
	}
	if driver[0] < 0 {
		return binpack.EmptyPackingResult(), true
	}
	res := &binpack.PackingResult{DriverNode: l.s.names[driver[0]], HasCapacity: true, ExecutorNodes: make([]string, executorCount)}
	for i := 0; i < executorCount; i++ {
		res.ExecutorNodes[i] = l.s.names[exec[i]]
	}
	res.PackingEfficiencies = efficienciesFor(md, driverResources, executorResources, res, true)
	return res, true
}

// RescheduleExecutorNode is the node choice of rescheduleExecutor (EXT/resource.go:652-662, 675-705) on the device:
// minFrag selects rescheduleExecutorWithMinimalFragmentation (`md` = availableNodesSchedulingMetadata of :640, `overhead`
// the map it hands to GetNodeCapacities, `hosting` = getNodesWithExecutorsBelongingToSameApp); otherwise the first
// node of the order that fits (`md` then carries availableResources of :643).  ok=false: run the Go code instead.
func RescheduleExecutorNode(minFrag bool, executorResources *resources.Resources, executorNodeNames []string,
	md resources.NodeGroupSchedulingMetadata, overhead resources.NodeGroupResources, hosting map[string]bool) (node string, found, ok bool) {
	d, err := getDevice()
	if err != nil {
		return "", false, false
	}
	ec, em, eg, ok1 := toTriple(executorResources)
	s, ok2 := marshal(md, nil, executorNodeNames)
	if !ok1 || !ok2 || len(s.names) == 0 {
		return "", false, ok1 && ok2
	}
	index := make(map[string]int32, len(s.names))
	for i, n := range s.names {
		index[n] = int32(i)
	}
	rc, rm, rg := make([]int64, len(s.names)), make([]int64, len(s.names)), make([]int64, len(s.names))
	hostNodes, hostOff := []int32{}, []int64{0, 0}
	in := C.gp_reschedule{n_execs: 1, exe_cpu_milli: (*C.int64_t)(unsafe.Pointer(&ec)), exe_mem_bytes: (*C.int64_t)(unsafe.Pointer(&em)),
		exe_gpu: (*C.int64_t)(unsafe.Pointer(&eg))}
	if minFrag {
		for n, r := range overhead {
			if i, known := index[n]; known {
				var exact bool
				if rc[i], rm[i], rg[i], exact = toTriple(r); !exact {
					return "", false, false
				}
			}
		}
		for n, yes := range hosting {
			if i, known := index[n]; known && yes {
				hostNodes = append(hostNodes, i)
			}
		}
		hostOff[1] = int64(len(hostNodes))
		in.min_frag = 1
		in.reserved_cpu_milli, in.reserved_mem_bytes, in.reserved_gpu = ptr64(rc), ptr64(rm), ptr64(rg)
		in.host_off, in.host_nodes = ptr64(hostOff), ptr32(hostNodes)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	if err := d.setSnapshot(s); err != nil {
		return "", false, false
	}
	var out C.int32_t = -1
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{&ec, &em, &eg, ptrOrNil(rc), ptrOrNil(rm), ptrOrNil(rg), &hostOff[0], ptrOrNil32(hostNodes)} {
		if p != nil {
			pin.Pin(p)
		}
	}
	if st := C.gp_reschedule_executors(d.ctx, &in, &out); st != C.GP_OK {
		return "", false, false
	}
	if out < 0 {
		return "", false, true // failureFit, :672
	}
	return s.names[out], true, true
}

// The two zone labels rescheduleExecutor reads, and they differ (SURVEY App. B5): PotentialNodes sorts by
// NodeSchedulingMetadata.ZoneLabel, the BETA label with the placeholder "default" when it is absent
// (LIB/resources/resources.go:27,78-81); filterNodesToZone and getAzsOfPods read the GA label (EXT/resource.go:466,526).
const (
	labelZoneFailureDomain = "failure-domain.beta.kubernetes.io/zone" // corev1.LabelZoneFailureDomain
	labelTopologyZone      = "topology.kubernetes.io/zone"            // v1.LabelTopologyZone
)

// RescheduleNode is one node of availableNodes (getNodes(nodeNames), EXT/resource.go:604) as rescheduleExecutor reads it.
type RescheduleNode struct {
	Name          string
	Allocatable   *resources.Resources // node.Status.Allocatable
	Labels        map[string]string    // node.Labels: both zone labels are read from here
	Unschedulable bool
	Ready         bool
	ExecutorRank  int32 // rank of the node's executor-prioritized-node-label value, -1 unknown
}

// ReservationRow is one hard or soft reservation (GetReservedResources, EXT/resourcereservations.go:258-263).
type ReservationRow struct {
	Node      string
	Resources *resources.Resources
}

// RescheduleExecutorFromReservations is the whole of rescheduleExecutor (EXT/resource.go:594-673) minus pod and lister I/O in
// ONE gp_reschedule_from_reservations call: the reservations, both availabilities, PotentialNodes' executor order and the
// first-fit / minimal-fragmentation choice stay on the device, and the resident driver snapshot is left alone.  commonZone:
// the zone getCommonZoneForExecutorsApplication returned, or nil.  labelRanked: executor-prioritized-node-label configured.
// ok=false (any non-OK status, an inexact quantity, or a choice the reference leaves to its unstable sort): run the Go code.
func RescheduleExecutorFromReservations(minFrag bool, executorResources *resources.Resources, nodes []RescheduleNode,
	reservations []ReservationRow, overhead resources.NodeGroupResources, labelRanked bool, commonZone *string,
	hosting map[string]bool) (node string, found, ok bool) {
	d, err := getDevice()
	if err != nil || len(nodes) == 0 {
		return "", false, false
	}
	ec, em, eg, exact := toTriple(executorResources)
	if !exact {
		return "", false, false
	}
	n := len(nodes)
	index := make(map[string]int32, n)
	zoneID, topoID := make(map[string]int32), make(map[string]int32) // sorter zones and topology zones, interned separately
	ac, am, ag := make([]int64, n), make([]int64, n), make([]int64, n)
	oc, om, og := make([]int64, n), make([]int64, n), make([]int64, n)
	zone, topo, nameRank, labelRank := make([]int32, n), make([]int32, n), make([]int32, n), make([]int32, n)
	unsched, ready := make([]uint8, n), make([]uint8, n)
	names := make([]string, n)
	for i, nd := range nodes {
		index[nd.Name] = int32(i)
		names[i] = nd.Name
		if ac[i], am[i], ag[i], exact = toTriple(nd.Allocatable); !exact {
			return "", false, false
		}
		if o, has := overhead[nd.Name]; has {
			if oc[i], om[i], og[i], exact = toTriple(o); !exact {
				return "", false, false
			}
		}
		sortZone, has := nd.Labels[labelZoneFailureDomain] // NodeSchedulingMetadataForNodes, resources.go:78-81
		if !has {
			sortZone = "default"
		}
		z, seen := zoneID[sortZone]
		if !seen {
			z = int32(len(zoneID))
			zoneID[sortZone] = z
		}
		zone[i], topo[i] = z, -1
		if ga, has := nd.Labels[labelTopologyZone]; has { // filterNodesToZone, EXT/resource.go:466
			t, seen := topoID[ga]
			if !seen {
				t = int32(len(topoID))
				topoID[ga] = t
			}
			topo[i] = t
		}
		if nd.Unschedulable {
			unsched[i] = 1
		}
		if nd.Ready {
			ready[i] = 1
		}
		labelRank[i] = nd.ExecutorRank
	}
	byName := make([]int32, n)
	for i := range byName {
		byName[i] = int32(i)
	}
	sort.Slice(byName, func(a, b int) bool { return names[byName[a]] < names[byName[b]] })
	for r, i := range byName {
		nameRank[i] = int32(r)
	}
	R := len(reservations)
	rn, rc, rm, rg := make([]int32, R), make([]int64, R), make([]int64, R), make([]int64, R)
	for t, r := range reservations {
		rn[t] = -1 // a reservation on a node outside the table is ignored (LIB/resources/resources.go:72-75)
		if i, known := index[r.Node]; known {
			rn[t] = i
		}
		if rc[t], rm[t], rg[t], exact = toTriple(r.Resources); !exact {
			return "", false, false
		}
	}
	hostNodes, hostOff := []int32{}, []int64{0, 0}
	for h, yes := range hosting {
		if i, known := index[h]; known && yes {
			hostNodes = append(hostNodes, i)
		}
	}
	hostOff[1] = int64(len(hostNodes))
	u := C.gp_usage_input{n_nodes: C.int32_t(n), alloc_cpu_milli: ptr64(ac), alloc_mem_bytes: ptr64(am), alloc_gpu: ptr64(ag),
		overhead_cpu_milli: ptr64(oc), overhead_mem_bytes: ptr64(om), overhead_gpu: ptr64(og), n_reservations: C.int64_t(R),
		res_node: ptr32(rn), res_cpu_milli: ptr64(rc), res_mem_bytes: ptr64(rm), res_gpu: ptr64(rg)}
	s := C.gp_sort_input{n_nodes: C.int32_t(n), n_zones: C.int32_t(len(zoneID)), zone_id: ptr32(zone), name_rank: ptr32(nameRank),
		unschedulable: ptr8(unsched), ready: ptr8(ready)}
	if labelRanked {
		s.executor_label_rank = ptr32(labelRank)
	}
	scope := C.gp_reschedule_scope{keep_topology_zone: -1, topology_zone: ptr32(topo)}
	var scopeArg *C.gp_reschedule_scope
	if commonZone != nil {
		scope.keep_topology_zone = C.int32_t(len(topoID)) // a zone no node carries: nothing is kept
		if z, seen := topoID[*commonZone]; seen {
			scope.keep_topology_zone = C.int32_t(z)
		}
		scopeArg = &scope
	}
	in := C.gp_reschedule{n_execs: 1, exe_cpu_milli: (*C.int64_t)(unsafe.Pointer(&ec)), exe_mem_bytes: (*C.int64_t)(unsafe.Pointer(&em)),
		exe_gpu: (*C.int64_t)(unsafe.Pointer(&eg))}
	if minFrag {
		in.min_frag = 1
		in.host_off, in.host_nodes = ptr64(hostOff), ptr32(hostNodes)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var out C.int32_t = -1
	var ambiguous C.uint8_t
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{&ec, &em, &eg, &hostOff[0], ptrOrNil32(hostNodes), ptrOrNil(ac), ptrOrNil(am), ptrOrNil(ag), ptrOrNil(oc),
		ptrOrNil(om), ptrOrNil(og), ptrOrNil32(rn), ptrOrNil(rc), ptrOrNil(rm), ptrOrNil(rg), ptrOrNil32(zone), ptrOrNil32(topo),
		ptrOrNil32(nameRank), ptrOrNil32(labelRank), ptrOrNil8(unsched), ptrOrNil8(ready)} {
		if p != nil {
			pin.Pin(p)
		}
	}
	if st := C.gp_reschedule_from_reservations(d.ctx, &u, &s, scopeArg, &in, &out, &ambiguous); st != C.GP_OK || ambiguous != 0 {
		return "", false, false // a missing zone label under a scope is refused here too: the Go code returns filterNodesToZone's error
	}
	if out < 0 {
		return "", false, true // failureFit, :672
	}
	return names[out], true, true
}

// QueuedApp is what fitEarlierDrivers reads from one earlier driver pod (EXT/resource.go:230-243).
type QueuedApp struct {
	Driver, Executor *resources.Resources
	MinExecutorCount int
	SkipIfNoFit      bool // shouldSkipDriverFifo (EXT/resource.go:264-270)
}

// FitEarlierDriversBatch replaces the body of fitEarlierDrivers (EXT/resource.go:224-262): ONE cgo call
// packs the whole queue in order on the device against the mutating snapshot (GP_MODE_FIFO_REFERENCE keeps
// the sparkResourceUsage accounting, EXT/sparkpods.go:139-146) and writes the charged availability back
// into metadata, as SubtractUsageIfExists (LIB/resources/resources.go:129-135) would have.
// ok=false: the caller must run the original Go loop instead.
func FitEarlierDriversBatch(algo C.gp_algo, apps []QueuedApp, nodeNames, executorNodeNames []string,
	metadata resources.NodeGroupSchedulingMetadata) (fits bool, ok bool) {
	d, err := getDevice()
	if err != nil {
		return false, false
	}
	if len(apps) == 0 {
		return true, true // no earlier drivers: nothing to fit, nothing to subtract (EXT/resource.go:230 loop body never runs)
	}
	s, exact := marshal(metadata, nodeNames, executorNodeNames)
	if !exact {
		return false, false
	}
	q := len(apps)
	dc, dm, dg := make([]int64, q), make([]int64, q), make([]int64, q)
	ec, em, eg := make([]int64, q), make([]int64, q), make([]int64, q)
	cnt, skip, off := make([]int32, q), make([]uint8, q), make([]int64, q+1)
	for i, a := range apps {
		var o1, o2 bool
		dc[i], dm[i], dg[i], o1 = toTriple(a.Driver)
		ec[i], em[i], eg[i], o2 = toTriple(a.Executor)
		if !o1 || !o2 || a.MinExecutorCount < 0 {
			return false, false
		}
		cnt[i] = int32(a.MinExecutorCount)
		if a.SkipIfNoFit {
			skip[i] = 1
		}
		off[i+1] = off[i] + int64(cnt[i])
	}
	driver := make([]int32, q)
	exec := make([]int32, max(int(off[q]), 1))
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	if err := d.setSnapshot(s); err != nil {
		return false, false
	}
	// gp_apps / gp_results hold Go pointers: every slice base is pinned for the duration of the call
	// (cgocheck: "Go pointer to unpinned Go pointer"), exactly as setSnapshot does for the node table.
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{ptrOrNil(dc), ptrOrNil(dm), ptrOrNil(dg), ptrOrNil(ec), ptrOrNil(em), ptrOrNil(eg),
		ptrOrNil32(cnt), ptrOrNil8(skip), ptrOrNil(off), ptrOrNil32(driver), ptrOrNil32(exec)} {
		if p != nil {
			pin.Pin(p)
		}
	}
	ga := C.gp_apps{n_apps: C.int32_t(q), drv_cpu_milli: ptr64(dc), drv_mem_bytes: ptr64(dm), drv_gpu: ptr64(dg),
		exe_cpu_milli: ptr64(ec), exe_mem_bytes: ptr64(em), exe_gpu: ptr64(eg), exe_count: ptr32(cnt),
		skip_if_no_fit: ptr8(skip), exec_out_off: ptr64(off)}
	gr := C.gp_results{driver_node: ptr32(driver), executor_nodes: ptr32(exec), executor_nodes_cap: C.int64_t(len(exec))}
	if st := C.gp_pack_batch(d.ctx, &ga, algo, C.GP_MODE_FIFO_REFERENCE, &gr); st != C.GP_OK {
		return false, false
	}
	cpu, mem, gpu := make([]int64, len(s.names)), make([]int64, len(s.names)), make([]int64, len(s.names))
	if st := C.gp_get_snapshot(d.ctx, ptr64(cpu), ptr64(mem), ptr64(gpu)); st != C.GP_OK {
		return false, false
	}
	for i, n := range s.names {
		a := metadata[n].AvailableResources
		a.CPU = *resource.NewMilliQuantity(cpu[i], resource.DecimalSI)
		a.Memory = *resource.NewQuantity(mem[i], resource.BinarySI)
		a.NvidiaGPU = *resource.NewQuantity(gpu[i], resource.DecimalSI)
	}
	fits = true
	for i := range apps {
		if driver[i] == -2 || (driver[i] == -1 && skip[i] == 0) {
			fits = false
		}
	}
	return fits, true
}

// FitEarlierDriversSingleAZ is FitEarlierDriversBatch for `binpack: single-az-tightly-pack` (algo GP_TIGHTLY_PACK) and
// `single-az-minimal-fragmentation` (algo GP_MINIMAL_FRAGMENTATION): fitEarlierDrivers (EXT/resource.go:224-262) when
// binpacker.BinpackFunc packs every zone and keeps the best result (LIB/binpack/single_az.go:23-97).  The zones of
// groupNodesByZone (:57-73) become the snapshot's instance groups, SchedulableResources go up with gp_set_schedulable, and
// ONE gp_pack_fifo_zones call runs the whole queue on the device -- the zone chosen for driver i feeds driver i+1 there.
// ok=false: the caller must run the original Go loop instead.
func FitEarlierDriversSingleAZ(algo C.gp_algo, apps []QueuedApp, nodeNames, executorNodeNames []string,
	metadata resources.NodeGroupSchedulingMetadata) (fits bool, ok bool) {
	d, err := getDevice()
	if err != nil {
		return false, false
	}
	if len(apps) == 0 {
		return true, true
	}
	// groupNodesByZone for both orders; zones without executor candidates are left out (single_az.go:38-41)
	group := func(names []string) ([]string, map[string][]string) {
		order, byZone := []string{}, map[string][]string{}
		for _, n := range names {
			m, present := metadata[n]
			if !present {
				continue
			}
			if _, seen := byZone[m.ZoneLabel]; !seen {
				order = append(order, m.ZoneLabel)
			}
			byZone[m.ZoneLabel] = append(byZone[m.ZoneLabel], n)
		}
		return order, byZone
	}
	zones, dz := group(nodeNames)
	_, ez := group(executorNodeNames)
	s := &snapshot{}
	index := map[string]int32{}
	var sc, sm, sg []int64
	intern := func(n string) (int32, bool) {
		if i, seen := index[n]; seen {
			return i, true
		}
		m := metadata[n]
		c, mm, g, exact := toTriple(m.AvailableResources)
		c2, m2, g2, exact2 := toTriple(m.SchedulableResources)
		if !exact || !exact2 {
			return -1, false
		}
		i := int32(len(s.names))
		index[n] = i
		s.names = append(s.names, n)
		s.cpu, s.mem, s.gpu = append(s.cpu, c), append(s.mem, mm), append(s.gpu, g)
		sc, sm, sg = append(sc, c2), append(sm, m2), append(sg, g2)
		return i, true
	}
	eoff, doff := []int32{0}, []int32{0}
	for _, z := range zones {
		eo, has := ez[z]
		if !has {
			continue
		}
		for _, n := range eo {
			i, exact := intern(n)
			if !exact {
				return false, false
			}
			s.execIdx = append(s.execIdx, i)
		}
		for _, n := range dz[z] {
			i, exact := intern(n)
			if !exact {
				return false, false
			}
			s.drvIdx = append(s.drvIdx, i)
		}
		eoff, doff = append(eoff, int32(len(s.execIdx))), append(doff, int32(len(s.drvIdx)))
	}
	nGroups := len(eoff) - 1
	if nGroups == 0 || nGroups > 64 {
		return false, false // no candidate zone (every BinpackFunc call is an EmptyPackingResult) or too many: the Go loop decides
	}
	q := len(apps)
	dc, dm, dg := make([]int64, q), make([]int64, q), make([]int64, q)
	ec, em, eg := make([]int64, q), make([]int64, q), make([]int64, q)
	cnt, skip := make([]int32, q), make([]uint8, q)
	total := 0
	for i, a := range apps {
		var o1, o2 bool
		dc[i], dm[i], dg[i], o1 = toTriple(a.Driver)
		ec[i], em[i], eg[i], o2 = toTriple(a.Executor)
		if !o1 || !o2 || a.MinExecutorCount < 0 {
			return false, false
		}
		cnt[i] = int32(a.MinExecutorCount)
		if a.SkipIfNoFit {
			skip[i] = 1
		}
		total += a.MinExecutorCount
	}
	zone, driver := make([]int32, q), make([]int32, q)
	exec := make([]int32, max(total, 1))
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{ptrOrNil(s.cpu), ptrOrNil(s.mem), ptrOrNil(s.gpu), ptrOrNil32(s.execIdx), ptrOrNil32(s.drvIdx),
		ptrOrNil32(eoff), ptrOrNil32(doff), ptrOrNil(sc), ptrOrNil(sm), ptrOrNil(sg),
		ptrOrNil(dc), ptrOrNil(dm), ptrOrNil(dg), ptrOrNil(ec), ptrOrNil(em), ptrOrNil(eg),
		ptrOrNil32(cnt), ptrOrNil8(skip), ptrOrNil32(zone), ptrOrNil32(driver), ptrOrNil32(exec)} {
		if p != nil {
			pin.Pin(p)
		}
	}
	gn := C.gp_nodes{
		n_nodes: C.int32_t(len(s.names)), avail_cpu_milli: ptr64(s.cpu), avail_mem_bytes: ptr64(s.mem), avail_gpu: ptr64(s.gpu),
		n_groups: C.int32_t(nGroups), exec_off: ptr32(eoff), exec_order: ptr32(s.execIdx), drv_off: ptr32(doff), drv_order: ptr32(s.drvIdx),
	}
	if st := C.gp_set_snapshot(d.ctx, &gn); st != C.GP_OK {
		return false, false
	}
	if st := C.gp_set_schedulable(d.ctx, ptr64(sc), ptr64(sm), ptr64(sg)); st != C.GP_OK {
		return false, false
	}
	ga := C.gp_apps{n_apps: C.int32_t(q), drv_cpu_milli: ptr64(dc), drv_mem_bytes: ptr64(dm), drv_gpu: ptr64(dg),
		exe_cpu_milli: ptr64(ec), exe_mem_bytes: ptr64(em), exe_gpu: ptr64(eg), exe_count: ptr32(cnt), skip_if_no_fit: ptr8(skip)}
	gz := C.gp_zone_results{zone: ptr32(zone), driver_node: ptr32(driver), executor_nodes: ptr32(exec), executor_nodes_cap: C.int64_t(len(exec))}
	if st := C.gp_pack_fifo_zones(d.ctx, &ga, algo, C.GP_MODE_FIFO_REFERENCE, &gz); st != C.GP_OK {
		return false, false
	}
	cpu, mem, gpu := make([]int64, len(s.names)), make([]int64, len(s.names)), make([]int64, len(s.names))
	if st := C.gp_get_snapshot(d.ctx, ptr64(cpu), ptr64(mem), ptr64(gpu)); st != C.GP_OK {
		return false, false
	}
	for i, n := range s.names { // SubtractUsageIfExists (LIB/resources/resources.go:129-135), as the device left it
		a := metadata[n].AvailableResources
		a.CPU = *resource.NewMilliQuantity(cpu[i], resource.DecimalSI)
		a.Memory = *resource.NewQuantity(mem[i], resource.BinarySI)
		a.NvidiaGPU = *resource.NewQuantity(gpu[i], resource.DecimalSI)
	}
	fits = true
	for i := range apps {
		if driver[i] == -2 || (driver[i] == -1 && skip[i] == 0) { // EXT/resource.go:250-252
			fits = false
		}
	}
	return fits, true
}

// azLayout is the snapshot of az-aware-tightly-pack (gp_pack_batch_az_aware, gp_pack_fifo_az_aware): the candidate zones
// become instance groups 0..nZones-1 (groupNodesByZone in driverZonesInOrder order, zones without executor candidates
// left out, single_az.go:36-41), one trailing group holds the other nodes of the two orders (a zone with driver candidates
// only, executor candidates of a zone without driver candidates), and the undivided orders go along as node indices of
// the same table (ue, ud).  sc / sm / sg: SchedulableResources of the table's nodes.
type azLayout struct {
	s                  *snapshot
	sc, sm, sg         []int64
	eoff, doff, ue, ud []int32
	nZones             int
}

// azAwareLayout marshals the layout; ok=false when a quantity is not an exact int64.
func azAwareLayout(nodeNames, executorNodeNames []string, metadata resources.NodeGroupSchedulingMetadata) (*azLayout, bool) {
	group := func(names []string) ([]string, map[string][]string) {
		order, byZone := []string{}, map[string][]string{}
		for _, n := range names {
			m, present := metadata[n]
			if !present {
				continue
			}
			if _, seen := byZone[m.ZoneLabel]; !seen {
				order = append(order, m.ZoneLabel)
			}
			byZone[m.ZoneLabel] = append(byZone[m.ZoneLabel], n)
		}
		return order, byZone
	}
	zones, dz := group(nodeNames)
	_, ez := group(executorNodeNames)
	l := &azLayout{s: &snapshot{}, eoff: []int32{0}, doff: []int32{0}}
	s := l.s
	index := map[string]int32{}
	intern := func(n string) (int32, bool) {
		if i, seen := index[n]; seen {
			return i, true
		}
		m := metadata[n]
		c, mm, g, exact := toTriple(m.AvailableResources)
		c2, m2, g2, exact2 := toTriple(m.SchedulableResources)
		if !exact || !exact2 {
			return -1, false
		}
		i := int32(len(s.names))
		index[n] = i
		s.names = append(s.names, n)
		s.cpu, s.mem, s.gpu = append(s.cpu, c), append(s.mem, mm), append(s.gpu, g)
		l.sc, l.sm, l.sg = append(l.sc, c2), append(l.sm, m2), append(l.sg, g2)
		return i, true
	}
	candidate := map[string]bool{}
	for _, z := range zones {
		eo, has := ez[z]
		if !has {
			continue
		}
		candidate[z] = true
		for _, n := range eo {
			i, exact := intern(n)
			if !exact {
				return nil, false
			}
			s.execIdx = append(s.execIdx, i)
		}
		for _, n := range dz[z] {
			i, exact := intern(n)
			if !exact {
				return nil, false
			}
			s.drvIdx = append(s.drvIdx, i)
		}
		l.eoff, l.doff = append(l.eoff, int32(len(s.execIdx))), append(l.doff, int32(len(s.drvIdx)))
	}
	l.nZones = len(l.eoff) - 1
	// the trailing group: every node of the two orders outside the candidate zones (only the fallback reaches it)
	rest := func(names []string, dst *[]int32) bool {
		for _, n := range names {
			m, present := metadata[n]
			if !present || candidate[m.ZoneLabel] {
				continue
			}
			i, exact := intern(n)
			if !exact {
				return false
			}
			*dst = append(*dst, i)
		}
		return true
	}
	if !rest(executorNodeNames, &s.execIdx) || !rest(nodeNames, &s.drvIdx) {
		return nil, false
	}
	if l.nZones == 0 || int(l.eoff[l.nZones]) < len(s.execIdx) || int(l.doff[l.nZones]) < len(s.drvIdx) {
		l.eoff, l.doff = append(l.eoff, int32(len(s.execIdx))), append(l.doff, int32(len(s.drvIdx)))
	}
	// the undivided orders (names absent from the metadata dropped)
	undivided := func(names []string) []int32 {
		out := make([]int32, 0, len(names))
		for _, n := range names {
			if i, seen := index[n]; seen {
				out = append(out, i)
			}
		}
		return out
	}
	l.ue, l.ud = undivided(executorNodeNames), undivided(nodeNames)
	return l, true
}

// pin keeps the layout's arrays in place while C holds pointers to them.
func (l *azLayout) pin(pin *runtime.Pinner) {
	for _, p := range []any{ptrOrNil(l.s.cpu), ptrOrNil(l.s.mem), ptrOrNil(l.s.gpu), ptrOrNil32(l.s.execIdx), ptrOrNil32(l.s.drvIdx),
		ptrOrNil32(l.eoff), ptrOrNil32(l.doff), ptrOrNil(l.sc), ptrOrNil(l.sm), ptrOrNil(l.sg), ptrOrNil32(l.ue), ptrOrNil32(l.ud)} {
		if p != nil {
			pin.Pin(p)
		}
	}
}

// upload sets the snapshot and its SchedulableResources on the device (d.mu held, arrays pinned).
func (l *azLayout) upload(d *device) bool {
	gn := C.gp_nodes{
		n_nodes: C.int32_t(len(l.s.names)), avail_cpu_milli: ptr64(l.s.cpu), avail_mem_bytes: ptr64(l.s.mem), avail_gpu: ptr64(l.s.gpu),
		n_groups: C.int32_t(len(l.eoff) - 1), exec_off: ptr32(l.eoff), exec_order: ptr32(l.s.execIdx), drv_off: ptr32(l.doff),
		drv_order: ptr32(l.s.drvIdx),
	}
	if st := C.gp_set_snapshot(d.ctx, &gn); st != C.GP_OK {
		return false
	}
	return C.gp_set_schedulable(d.ctx, ptr64(l.sc), ptr64(l.sm), ptr64(l.sg)) == C.GP_OK
}

func (l *azLayout) orders() C.gp_az_orders {
	return C.gp_az_orders{n_zones: C.int32_t(l.nZones), n_exec: C.int32_t(len(l.ue)), exec_order: ptr32(l.ue),
		n_drv: C.int32_t(len(l.ud)), drv_order: ptr32(l.ud)}
}

// FitEarlierDriversAzAware is FitEarlierDriversSingleAZ for `binpack: az-aware-tightly-pack` (AzAwareTightlyPack,
// LIB/binpack/az_aware_pack_tightly.go:27-38) on the az-aware layout (azAwareLayout).  ONE gp_pack_fifo_az_aware call
// runs the whole queue: the zone packs, and when no zone wins the fallback over the undivided orders, both on the device.
// ok=false: the caller must run the original Go loop instead (also above 64 candidate zones).
func FitEarlierDriversAzAware(apps []QueuedApp, nodeNames, executorNodeNames []string,
	metadata resources.NodeGroupSchedulingMetadata) (fits bool, ok bool) {
	d, err := getDevice()
	if err != nil {
		return false, false
	}
	if len(apps) == 0 {
		return true, true
	}
	l, exact := azAwareLayout(nodeNames, executorNodeNames, metadata)
	if !exact || l.nZones > 64 {
		return false, false // gp_pack_fifo_az_aware takes at most 64 candidate zones: the Go loop decides
	}
	s := l.s
	q := len(apps)
	dc, dm, dg := make([]int64, q), make([]int64, q), make([]int64, q)
	ec, em, eg := make([]int64, q), make([]int64, q), make([]int64, q)
	cnt, skip := make([]int32, q), make([]uint8, q)
	total := 0
	for i, a := range apps {
		var o1, o2 bool
		dc[i], dm[i], dg[i], o1 = toTriple(a.Driver)
		ec[i], em[i], eg[i], o2 = toTriple(a.Executor)
		if !o1 || !o2 || a.MinExecutorCount < 0 {
			return false, false
		}
		cnt[i] = int32(a.MinExecutorCount)
		if a.SkipIfNoFit {
			skip[i] = 1
		}
		total += a.MinExecutorCount
	}
	zone, driver := make([]int32, q), make([]int32, q)
	exec := make([]int32, max(total, 1))
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	l.pin(&pin)
	for _, p := range []any{ptrOrNil(dc), ptrOrNil(dm), ptrOrNil(dg), ptrOrNil(ec), ptrOrNil(em), ptrOrNil(eg),
		ptrOrNil32(cnt), ptrOrNil8(skip), ptrOrNil32(zone), ptrOrNil32(driver), ptrOrNil32(exec)} {
		if p != nil {
			pin.Pin(p)
		}
	}
	if !l.upload(d) {
		return false, false
	}
	ga := C.gp_apps{n_apps: C.int32_t(q), drv_cpu_milli: ptr64(dc), drv_mem_bytes: ptr64(dm), drv_gpu: ptr64(dg),
		exe_cpu_milli: ptr64(ec), exe_mem_bytes: ptr64(em), exe_gpu: ptr64(eg), exe_count: ptr32(cnt), skip_if_no_fit: ptr8(skip)}
	orders := l.orders()
	gz := C.gp_zone_results{zone: ptr32(zone), driver_node: ptr32(driver), executor_nodes: ptr32(exec), executor_nodes_cap: C.int64_t(len(exec))}
	if st := C.gp_pack_fifo_az_aware(d.ctx, &ga, C.GP_MODE_FIFO_REFERENCE, &orders, &gz); st != C.GP_OK {
		return false, false
	}
	cpu, mem, gpu := make([]int64, len(s.names)), make([]int64, len(s.names)), make([]int64, len(s.names))
	if st := C.gp_get_snapshot(d.ctx, ptr64(cpu), ptr64(mem), ptr64(gpu)); st != C.GP_OK {
		return false, false
	}
	for i, n := range s.names { // SubtractUsageIfExists (LIB/resources/resources.go:129-135), as the device left it
		a := metadata[n].AvailableResources
		a.CPU = *resource.NewMilliQuantity(cpu[i], resource.DecimalSI)
		a.Memory = *resource.NewQuantity(mem[i], resource.BinarySI)
		a.NvidiaGPU = *resource.NewQuantity(gpu[i], resource.DecimalSI)
	}
	fits = true
	for i := range apps {
		if driver[i] == -2 || (driver[i] == -1 && skip[i] == 0) { // EXT/resource.go:250-252
			fits = false
		}
	}
	return fits, true
}

// gpBinpacker maps a `binpack:` value to the device packer; unknown names select distribute-evenly, like SelectBinpacker
// (internal/binpacker/binpack.go:52-58).
func gpBinpacker(name string) C.gp_binpacker {
	switch name {
	case "tightly-pack":
		return C.GP_BP_TIGHTLY_PACK
	case "az-aware-tightly-pack":
		return C.GP_BP_AZ_AWARE_TIGHTLY_PACK
	case "single-az-tightly-pack":
		return C.GP_BP_SINGLE_AZ_TIGHTLY_PACK
	case "single-az-minimal-fragmentation":
		return C.GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION
	}
	return C.GP_BP_DISTRIBUTE_EVENLY
}

// StaleDriver is one driver the unschedulable-pod marker checks (scanForUnschedulablePods, EXT/unschedulablepods.go:93-129):
// its application resources and its required node affinity, an index into the distinct affinities of the sweep.
type StaleDriver struct {
	DriverResources, ExecutorResources *resources.Resources
	MinExecutorCount                   int
	Affinity                           int32
}

// NodeAffinity is one distinct required node affinity: what GetRequiredNodeAffinity(pod) reads
// (K8S/component-helpers/scheduling/corev1/nodeaffinity/nodeaffinity.go:297-324).
type NodeAffinity struct {
	NodeSelector map[string]string
	Required     *v1.NodeSelector // pod.Spec.Affinity.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution; nil = none
}

// RequiredNodeAffinityOf reads a pod's NodeAffinity.
func RequiredNodeAffinityOf(pod *v1.Pod) NodeAffinity {
	a := NodeAffinity{NodeSelector: pod.Spec.NodeSelector}
	if pod.Spec.Affinity != nil && pod.Spec.Affinity.NodeAffinity != nil {
		a.Required = pod.Spec.Affinity.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution
	}
	return a
}

// affinityArrays holds gp_node_labels and gp_node_affinities.  Label keys and values become dense ids; every rule that needs
// the strings is applied here with the reference's own functions: labels.NewRequirement (the operator mapping of
// nodeSelectorRequirementsAsSelector, nodeaffinity.go:203-241) and the In / NotIn-with-one-value rule of
// nodeSelectorRequirementsAsFieldSelector (:248-280) set a term's parse_error flag, strconv.ParseInt(v, 10, 64) gives
// label_int_ok / label_int, metadata.name becomes a node index (-1: no such node) and any other field key, which reads ""
// (extractNodeFields), a constant requirement.  The same rules as affinity.encode() in the Python package.
type affinityArrays struct {
	nKeys, nValues                                          int32
	labelOff, labelInt, selOff, termOff, termReqOff         []int64
	reqInt, reqValOff                                       []int64
	labelKey, labelVal, selKey, selVal, reqOp, reqKey, reqVal []int32
	labelIntOK, hasRequired, termParseError                 []uint8
}

var labelOps = map[v1.NodeSelectorOperator]struct {
	sel selection.Operator
	op  C.int32_t
}{
	v1.NodeSelectorOpIn: {selection.In, C.GP_AFF_IN}, v1.NodeSelectorOpNotIn: {selection.NotIn, C.GP_AFF_NOT_IN},
	v1.NodeSelectorOpExists: {selection.Exists, C.GP_AFF_EXISTS}, v1.NodeSelectorOpDoesNotExist: {selection.DoesNotExist, C.GP_AFF_DOES_NOT_EXIST},
	v1.NodeSelectorOpGt: {selection.GreaterThan, C.GP_AFF_GT}, v1.NodeSelectorOpLt: {selection.LessThan, C.GP_AFF_LT},
}

func internAffinities(nodes []*v1.Node, affinities []NodeAffinity) *affinityArrays {
	e := &affinityArrays{labelOff: []int64{0}, selOff: []int64{0}, termOff: []int64{0}, termReqOff: []int64{0}, reqValOff: []int64{0}}
	keys, vals, nodeIndex := map[string]int32{}, map[string]int32{}, map[string]int64{}
	id := func(m map[string]int32, s string) int32 {
		v, seen := m[s]
		if !seen {
			v = int32(len(m))
			m[s] = v
		}
		return v
	}
	for i, n := range nodes {
		nodeIndex[n.Name] = int64(i)
	}
	for _, n := range nodes {
		type ent struct {
			k int32
			v string
		}
		ents := make([]ent, 0, len(n.Labels))
		for k, v := range n.Labels {
			ents = append(ents, ent{id(keys, k), v})
		}
		sort.Slice(ents, func(a, b int) bool { return ents[a].k < ents[b].k })
		for _, en := range ents {
			iv, err := strconv.ParseInt(en.v, 10, 64)
			ok := uint8(0)
			if err == nil {
				ok = 1
			} else {
				iv = 0
			}
			e.labelKey, e.labelVal = append(e.labelKey, en.k), append(e.labelVal, id(vals, en.v))
			e.labelIntOK, e.labelInt = append(e.labelIntOK, ok), append(e.labelInt, iv)
		}
		e.labelOff = append(e.labelOff, int64(len(e.labelKey)))
	}
	addReq := func(op C.int32_t, key int32, bound int64, vs []int32) {
		sort.Slice(vs, func(a, b int) bool { return vs[a] < vs[b] })
		e.reqOp, e.reqKey, e.reqInt = append(e.reqOp, int32(op)), append(e.reqKey, key), append(e.reqInt, bound)
		for j, v := range vs {
			if j == 0 || v != vs[j-1] {
				e.reqVal = append(e.reqVal, v)
			}
		}
		e.reqValOff = append(e.reqValOff, int64(len(e.reqVal)))
	}
	for _, a := range affinities {
		for k, v := range a.NodeSelector {
			e.selKey, e.selVal = append(e.selKey, id(keys, k)), append(e.selVal, id(vals, v))
		}
		e.selOff = append(e.selOff, int64(len(e.selKey)))
		has := uint8(0)
		var terms []v1.NodeSelectorTerm
		if a.Required != nil {
			has, terms = 1, a.Required.NodeSelectorTerms
		}
		e.hasRequired = append(e.hasRequired, has)
		for _, t := range terms {
			bad := false
			for _, r := range t.MatchExpressions {
				o, known := labelOps[r.Operator]
				if !known {
					bad = true
				} else if _, err := labels.NewRequirement(r.Key, o.sel, r.Values); err != nil {
					bad = true
				}
			}
			for _, r := range t.MatchFields {
				if (r.Operator != v1.NodeSelectorOpIn && r.Operator != v1.NodeSelectorOpNotIn) || len(r.Values) != 1 {
					bad = true
				}
			}
			flag := uint8(0)
			if bad {
				flag = 1
			} else {
				for _, r := range t.MatchExpressions {
					o := labelOps[r.Operator]
					var bound int64
					var vs []int32
					switch o.op {
					case C.GP_AFF_GT, C.GP_AFF_LT:
						bound, _ = strconv.ParseInt(r.Values[0], 10, 64)
					case C.GP_AFF_IN, C.GP_AFF_NOT_IN:
						for _, v := range r.Values {
							vs = append(vs, id(vals, v))
						}
					}
					addReq(o.op, id(keys, r.Key), bound, vs)
				}
				for _, r := range t.MatchFields {
					in := r.Operator == v1.NodeSelectorOpIn
					if r.Key == "metadata.name" {
						idx, found := nodeIndex[r.Values[0]]
						if !found {
							idx = -1
						}
						op := C.int32_t(C.GP_AFF_FIELD_NAME_NOT_IN)
						if in {
							op = C.GP_AFF_FIELD_NAME_IN
						}
						addReq(op, 0, idx, nil)
					} else if (r.Values[0] == "") == in { // any other field reads "": always true
						addReq(C.GP_AFF_FIELD_NAME_NOT_IN, 0, -1, nil)
					} else { // never true
						addReq(C.GP_AFF_FIELD_NAME_IN, 0, -1, nil)
					}
				}
			}
			e.termParseError = append(e.termParseError, flag)
			e.termReqOff = append(e.termReqOff, int64(len(e.reqOp)))
		}
		e.termOff = append(e.termOff, int64(len(e.termParseError)))
	}
	e.nKeys, e.nValues = int32(len(keys)), int32(len(vals))
	// one spare element each: no slice base is nil and every one can be pinned
	e.labelKey, e.labelVal, e.selKey, e.selVal = append(e.labelKey, 0), append(e.labelVal, 0), append(e.selKey, 0), append(e.selVal, 0)
	e.reqOp, e.reqKey, e.reqVal, e.labelInt, e.reqInt = append(e.reqOp, 0), append(e.reqKey, 0), append(e.reqVal, 0), append(e.labelInt, 0), append(e.reqInt, 0)
	e.labelIntOK, e.hasRequired, e.termParseError = append(e.labelIntOK, 0), append(e.hasRequired, 0), append(e.termParseError, 0)
	return e
}

// structs pins every slice base and returns the two C structs over them.
func (e *affinityArrays) structs(pin *runtime.Pinner, nNodes, nAff int) (C.gp_node_labels, C.gp_node_affinities) {
	for _, s := range [][]int64{e.labelOff, e.labelInt, e.selOff, e.termOff, e.termReqOff, e.reqInt, e.reqValOff} {
		pin.Pin(&s[0])
	}
	for _, s := range [][]int32{e.labelKey, e.labelVal, e.selKey, e.selVal, e.reqOp, e.reqKey, e.reqVal} {
		pin.Pin(&s[0])
	}
	for _, s := range [][]uint8{e.labelIntOK, e.hasRequired, e.termParseError} {
		pin.Pin(&s[0])
	}
	l := C.gp_node_labels{n_nodes: C.int32_t(nNodes), n_keys: C.int32_t(e.nKeys), n_values: C.int32_t(e.nValues),
		label_off: ptr64(e.labelOff), label_key: ptr32(e.labelKey), label_val: ptr32(e.labelVal), label_int_ok: ptr8(e.labelIntOK),
		label_int: ptr64(e.labelInt)}
	a := C.gp_node_affinities{n_aff: C.int32_t(nAff), sel_off: ptr64(e.selOff), sel_key: ptr32(e.selKey), sel_val: ptr32(e.selVal),
		has_required: ptr8(e.hasRequired), term_off: ptr64(e.termOff), term_req_off: ptr64(e.termReqOff),
		term_parse_error: ptr8(e.termParseError), req_op: ptr32(e.reqOp), req_key: ptr32(e.reqKey), req_int: ptr64(e.reqInt),
		req_val_off: ptr64(e.reqValOff), req_val: ptr32(e.reqVal)}
	return l, a
}

// MatchRequiredNodeAffinity is utils.ListWithPredicate(nodes, GetRequiredNodeAffinity(pod).Match) (internal/common/utils/
// pods.go:110-127) for every distinct affinity at once, in one gp_match_node_affinity call: selectDriverNode's
// availableNodes (EXT/resource.go:292-298).  matched[a] lists the nodes affinity a matches, in node order; failed[a] =
// some node gave an error -- ListWithPredicate's error, on which the Predicate fails with failureInternal.  ok=false (no
// device, any non-OK status): the caller runs ListWithPredicate in Go.
func MatchRequiredNodeAffinity(nodes []*v1.Node, affinities []NodeAffinity) (matched [][]*v1.Node, failed []bool, ok bool) {
	d, err := getDevice()
	if err != nil {
		return nil, nil, false
	}
	n, nAff := len(nodes), len(affinities)
	e := internAffinities(nodes, affinities)
	words := (n + 31) / 32
	member := make([]uint32, nAff*words+1)
	nMatch, nError := make([]int32, nAff+1), make([]int32, nAff+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	l, a := e.structs(&pin, n, nAff)
	pin.Pin(&member[0])
	pin.Pin(&nMatch[0])
	pin.Pin(&nError[0])
	out := C.gp_affinity_match{member: (*C.uint32_t)(unsafe.Pointer(&member[0])), n_match: ptr32(nMatch), n_error: ptr32(nError)}
	if C.gp_match_node_affinity(d.ctx, &l, &a, &out) != C.GP_OK {
		return nil, nil, false
	}
	matched, failed = make([][]*v1.Node, nAff), make([]bool, nAff)
	for p := 0; p < nAff; p++ {
		failed[p] = nError[p] > 0
		matched[p] = make([]*v1.Node, 0, nMatch[p])
		for i := 0; i < n; i++ {
			if member[p*words+i/32]>>(i%32)&1 != 0 {
				matched[p] = append(matched[p], nodes[i])
			}
		}
	}
	return matched, failed, true
}

// DoesPodsExceedClusterCapacity is DoesPodExceedClusterCapacity (EXT/unschedulablepods.go:132-166) for every stale driver of
// one marker sweep in ONE gp_exceeds_cluster_capacity_affinity call, whatever the `binpack:` value.  nodes is the node
// lister's list; nodesSchedulingMetadata is NodeSchedulingMetadataForNodes(nodes, zero usage, GetNonSchedulableOverhead):
// only SchedulableResources and ZoneLabel are read.  affinities holds each distinct required affinity of the stale drivers
// once and drivers[i].Affinity indexes it; the affinities' node sets may overlap freely.  affinityError[i]: the driver's
// affinity gave ListWithPredicate's error, on which the reference's scan returns (:113-117); exceeds[i] is then meaningless.
// The device context's resident snapshot is not touched.  ok=false (no device, an inexact quantity, a count outside int32,
// a node without metadata, any non-OK status): the caller runs DoesPodExceedClusterCapacity per driver in Go.
func DoesPodsExceedClusterCapacity(binpackerName string, nodes []*v1.Node, nodesSchedulingMetadata resources.NodeGroupSchedulingMetadata,
	affinities []NodeAffinity, drivers []StaleDriver) (exceeds, affinityError []bool, ok bool) {
	d, err := getDevice()
	if err != nil {
		return nil, nil, false
	}
	n, q := len(nodes), len(drivers)
	sc, sm, sg := make([]int64, n+1), make([]int64, n+1), make([]int64, n+1)
	zone := make([]int32, n+1)
	zoneID := map[string]int32{}
	for i, node := range nodes {
		md, found := nodesSchedulingMetadata[node.Name]
		if !found {
			return nil, nil, false
		}
		c, m, g, exact := toTriple(md.SchedulableResources)
		if !exact {
			return nil, nil, false
		}
		sc[i], sm[i], sg[i] = c, m, g
		z, seen := zoneID[md.ZoneLabel]
		if !seen {
			z = int32(len(zoneID))
			zoneID[md.ZoneLabel] = z
		}
		zone[i] = z
	}
	var cols [6][]int64
	for t := range cols {
		cols[t] = make([]int64, q+1)
	}
	count, prog := make([]int32, q+1), make([]int32, q+1)
	for j, drv := range drivers {
		dc, dm, dg, ok1 := toTriple(drv.DriverResources)
		ec, em, eg, ok2 := toTriple(drv.ExecutorResources)
		if !ok1 || !ok2 || drv.MinExecutorCount < 0 || drv.MinExecutorCount > math.MaxInt32 {
			return nil, nil, false
		}
		cols[0][j], cols[1][j], cols[2][j], cols[3][j], cols[4][j], cols[5][j] = dc, dm, dg, ec, em, eg
		count[j], prog[j] = int32(drv.MinExecutorCount), drv.Affinity
	}
	e := internAffinities(nodes, affinities)
	out, errs := make([]uint8, q+1), make([]uint8, q+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	// the C structs hold Go pointers: every slice base is pinned for the duration of the call
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{&sc[0], &sm[0], &sg[0], &zone[0], &count[0], &prog[0], &out[0], &errs[0]} {
		pin.Pin(p)
	}
	for t := range cols {
		pin.Pin(&cols[t][0])
	}
	l, a := e.structs(&pin, n, len(affinities))
	cn := C.gp_capacity_nodes{n_nodes: C.int32_t(n), alloc_cpu_milli: ptr64(sc), alloc_mem_bytes: ptr64(sm), alloc_gpu: ptr64(sg),
		n_zones: C.int32_t(max(len(zoneID), 1)), zone_id: ptr32(zone)}
	apps := C.gp_apps{n_apps: C.int32_t(q), drv_cpu_milli: ptr64(cols[0]), drv_mem_bytes: ptr64(cols[1]), drv_gpu: ptr64(cols[2]),
		exe_cpu_milli: ptr64(cols[3]), exe_mem_bytes: ptr64(cols[4]), exe_gpu: ptr64(cols[5]), exe_count: ptr32(count), group: ptr32(prog)}
	if C.gp_exceeds_cluster_capacity_affinity(d.ctx, &cn, &l, &a, &apps, gpBinpacker(binpackerName), ptr8(out), ptr8(errs)) != C.GP_OK {
		return nil, nil, false
	}
	exceeds, affinityError = make([]bool, q), make([]bool, q)
	for j := range exceeds {
		exceeds[j], affinityError[j] = out[j] != 0, errs[j] != 0
	}
	return exceeds, affinityError, true
}

// ReconcileNode is one lister node as the failover reconciler sees it (EXT/failover.go:286-314).
type ReconcileNode struct {
	Name             string
	Allocatable      *resources.Resources // from node.Status.Allocatable
	InstanceGroup    string               // n.Labels[instanceGroupLabel]; "" when the label is missing
	Unschedulable    bool                 // n.Spec.Unschedulable
	Ready            bool                 // NodeReady == True
	CreationUnixNano int64                // n.CreationTimestamp.UnixNano(): ordered like metav1.Time.Before
}

// ReconcileRow is one reservation of an RR, or one soft reservation: UsageForNodes + UsedSoftReservationResources (:315-317).
type ReconcileRow struct {
	Node      string
	Resources *resources.Resources
}

// ReconcileDriver is one stale driver, in the order its RR is written.
type ReconcileDriver struct {
	InstanceGroup     string // internal.FindInstanceGroupFromPodSpec
	ExecutorResources *resources.Resources
	MinExecutorCount  int
	RunningExecutors  int // len(sp.inconsistentExecutors); capped at MinExecutorCount as at :141-143
}

// ReconcileResult is what constructResourceReservation learns from findNodes for one driver.
type ReconcileResult struct {
	InstanceGroupFound bool     // false: "instance group not found" (:358-362), no RR and no charge
	ReservedNodeNames  []string // findNodes' result, possibly shorter than Min - running
}

// ReconcileFindNodes runs availableResourcesPerInstanceGroup and every stale driver's findNodes with the charge of :159 in one
// gp_reconcile_find_nodes call (DESIGN §2.3).  ok = false on any refusal or inexact quantity: the caller then runs the Go loop.
// The node slice is the lister's order; equal creation times keep it.
func ReconcileFindNodes(nodes []ReconcileNode, rows []ReconcileRow, overhead resources.NodeGroupResources, drivers []ReconcileDriver) ([]ReconcileResult, bool) {
	d, err := getDevice()
	if err != nil {
		return nil, false
	}
	n, r, q := len(nodes), len(rows), len(drivers)
	index := make(map[string]int32, n)
	groupID := map[string]int32{}
	intern := func(g string) int32 {
		id, seen := groupID[g]
		if !seen {
			id = int32(len(groupID))
			groupID[g] = id
		}
		return id
	}
	var al, ov [3][]int64
	for t := 0; t < 3; t++ {
		al[t], ov[t] = make([]int64, n+1), make([]int64, n+1)
	}
	grp, cre := make([]int32, n+1), make([]int64, n+1)
	unsched, ready := make([]uint8, n+1), make([]uint8, n+1)
	for i, nd := range nodes {
		index[nd.Name] = int32(i)
		var ok bool
		if al[0][i], al[1][i], al[2][i], ok = toTriple(nd.Allocatable); !ok {
			return nil, false
		}
		if o, in := overhead[nd.Name]; in {
			if ov[0][i], ov[1][i], ov[2][i], ok = toTriple(o); !ok {
				return nil, false
			}
		}
		grp[i], cre[i] = intern(nd.InstanceGroup), nd.CreationUnixNano
		if nd.Unschedulable {
			unsched[i] = 1
		}
		if nd.Ready {
			ready[i] = 1
		}
	}
	rn := make([]int32, r+1)
	var rc [3][]int64
	for t := 0; t < 3; t++ {
		rc[t] = make([]int64, r+1)
	}
	for j, row := range rows {
		rn[j] = -1 // a reservation on a node the lister no longer returns: AvailableForNodes never reads it
		if v, in := index[row.Node]; in {
			rn[j] = v
		}
		var ok bool
		if rc[0][j], rc[1][j], rc[2][j], ok = toTriple(row.Resources); !ok {
			return nil, false
		}
	}
	var ec [3][]int64
	for t := 0; t < 3; t++ {
		ec[t] = make([]int64, q+1)
	}
	count, dg, off := make([]int32, q+1), make([]int32, q+1), make([]int64, q+1)
	for j, drv := range drivers {
		var ok bool
		if ec[0][j], ec[1][j], ec[2][j], ok = toTriple(drv.ExecutorResources); !ok {
			return nil, false
		}
		k := drv.MinExecutorCount - min(drv.RunningExecutors, drv.MinExecutorCount) // :366
		if k < 0 {
			k = 0
		}
		if k > 1<<24 {
			return nil, false
		}
		count[j], dg[j] = int32(k), intern(drv.InstanceGroup)
		off[j+1] = off[j] + int64(k)
	}
	placed, exe := make([]int32, q+1), make([]int32, off[q]+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	// the C structs hold Go pointers: every slice base is pinned for the duration of the call
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []any{&grp[0], &cre[0], &unsched[0], &ready[0], &rn[0], &count[0], &dg[0], &off[0], &placed[0], &exe[0]} {
		pin.Pin(p)
	}
	for t := 0; t < 3; t++ {
		pin.Pin(&al[t][0])
		pin.Pin(&ov[t][0])
		pin.Pin(&rc[t][0])
		pin.Pin(&ec[t][0])
	}
	u := C.gp_usage_input{n_nodes: C.int32_t(n), alloc_cpu_milli: ptr64(al[0]), alloc_mem_bytes: ptr64(al[1]), alloc_gpu: ptr64(al[2]),
		overhead_cpu_milli: ptr64(ov[0]), overhead_mem_bytes: ptr64(ov[1]), overhead_gpu: ptr64(ov[2]),
		n_reservations: C.int64_t(r), res_node: ptr32(rn), res_cpu_milli: ptr64(rc[0]), res_mem_bytes: ptr64(rc[1]), res_gpu: ptr64(rc[2])}
	nd := C.gp_reconcile_nodes{n_groups: C.int32_t(max(len(groupID), 1)), node_group: ptr32(grp), creation: ptr64(cre),
		unschedulable: ptr8(unsched), ready: ptr8(ready)}
	a := C.gp_apps{n_apps: C.int32_t(q), exe_cpu_milli: ptr64(ec[0]), exe_mem_bytes: ptr64(ec[1]), exe_gpu: ptr64(ec[2]),
		exe_count: ptr32(count), group: ptr32(dg), exec_out_off: ptr64(off)}
	out := C.gp_reconcile_results{placed: ptr32(placed), executor_nodes: ptr32(exe), executor_nodes_cap: C.int64_t(off[q])}
	if C.gp_reconcile_find_nodes(d.ctx, &u, &nd, &a, &out) != C.GP_OK {
		return nil, false
	}
	res := make([]ReconcileResult, q)
	for j := range res {
		res[j].InstanceGroupFound = placed[j] >= 0
		for t := int32(0); t < placed[j]; t++ {
			res[j].ReservedNodeNames = append(res[j].ReservedNodeNames, nodes[exe[off[j]+int64(t)]].Name)
		}
	}
	return res, true
}

// ---- the overhead computer (internal/extender/overhead.go) ---------------------------------------------------------------

// OverheadRecords is the event side of the overhead computer kept as record slots for gp_node_overhead: register OnAdd,
// OnUpdate and OnDelete on the pod informer in place of NewOverheadComputer's handlers.  A slot per (node, UID) -- the
// reference's ClusterRequests map -- holds the pod's namespace, name and podToResources at its add event; deletes free the
// slot onto a free list.  Strings are interned once, when a record is written.
type OverheadRecords struct {
	mu       sync.Mutex
	at       map[[2]string]int // (nodeName, UID) -> slot
	free     []int
	ns       []string
	name     []string
	nodeID   []int32 // -1: free slot
	req      [3][]int64
	inexact  []bool // a quantity outside the exact-int64 model (sub-millicore cpu ...): every call falls back while one is held
	nInexact int
	nodeIx   map[string]int32
	nodes    []string
}

func NewOverheadRecords() *OverheadRecords {
	return &OverheadRecords{at: map[[2]string]int{}, nodeIx: map[string]int32{}}
}

func podToResources(pod *v1.Pod) *resources.Resources { // overhead.go:195-209
	res := resources.Zero()
	for _, c := range pod.Spec.Containers {
		res.AddFromResourceList(c.Resources.Requests)
	}
	for _, c := range pod.Spec.InitContainers {
		res.SetMaxResource(c.Resources.Requests)
	}
	return res
}

// OnAdd / OnUpdate / OnDelete: clientcache.FilteringResourceEventHandler{FilterFunc: spec.nodeName != ""} around
// addPodRequests / deletePodRequests -- the update that binds a pod is an add, the one that unbinds it a delete.
func (o *OverheadRecords) OnAdd(obj interface{}) {
	if pod, ok := obj.(*v1.Pod); ok && pod.Spec.NodeName != "" {
		o.record(pod)
	}
}

func (o *OverheadRecords) OnUpdate(oldObj, newObj interface{}) {
	oldPod, ok1 := oldObj.(*v1.Pod)
	newPod, ok2 := newObj.(*v1.Pod)
	if !ok1 || !ok2 {
		return
	}
	if newPod.Spec.NodeName != "" && oldPod.Spec.NodeName == "" {
		o.record(newPod)
	} else if newPod.Spec.NodeName == "" && oldPod.Spec.NodeName != "" {
		o.remove(oldPod)
	}
}

func (o *OverheadRecords) OnDelete(obj interface{}) {
	pod, ok := obj.(*v1.Pod)
	if !ok {
		if t, isTomb := obj.(clientcache.DeletedFinalStateUnknown); isTomb {
			pod, ok = t.Obj.(*v1.Pod)
		}
	}
	if ok && pod.Spec.NodeName != "" {
		o.remove(pod)
	}
}

func (o *OverheadRecords) record(pod *v1.Pod) {
	o.mu.Lock()
	defer o.mu.Unlock()
	key := [2]string{pod.Spec.NodeName, string(pod.UID)}
	i, ok := o.at[key]
	if !ok {
		if n := len(o.free); n > 0 {
			i, o.free = o.free[n-1], o.free[:n-1]
		} else {
			i = len(o.nodeID)
			o.ns, o.name, o.nodeID, o.inexact = append(o.ns, ""), append(o.name, ""), append(o.nodeID, -1), append(o.inexact, false)
			for d := range o.req {
				o.req[d] = append(o.req[d], 0)
			}
		}
		o.at[key] = i
	}
	id, known := o.nodeIx[pod.Spec.NodeName]
	if !known {
		id = int32(len(o.nodes))
		o.nodeIx[pod.Spec.NodeName] = id
		o.nodes = append(o.nodes, pod.Spec.NodeName)
	}
	cpu, mem, gpu, exact := toTriple(podToResources(pod))
	o.setInexact(i, !exact)
	o.ns[i], o.name[i], o.nodeID[i] = pod.Namespace, pod.Name, id
	o.req[0][i], o.req[1][i], o.req[2][i] = cpu, mem, gpu
}

func (o *OverheadRecords) remove(pod *v1.Pod) {
	o.mu.Lock()
	defer o.mu.Unlock()
	key := [2]string{pod.Spec.NodeName, string(pod.UID)}
	i, ok := o.at[key]
	if !ok {
		return
	}
	delete(o.at, key)
	o.setInexact(i, false)
	o.nodeID[i], o.ns[i], o.name[i] = -1, "", ""
	o.free = append(o.free, i)
}

func (o *OverheadRecords) setInexact(i int, v bool) {
	if o.inexact[i] != v {
		if v {
			o.nInexact++
		} else {
			o.nInexact--
		}
		o.inexact[i] = v
	}
}

// OverheadForNodes answers GetOverhead and GetNonSchedulableOverhead for `nodes` from one gp_node_overhead call: the
// driver and executor Predicates (EXT/resource.go:301, :639), the failover reconciler (failover.go:53) and the
// unschedulable marker (unschedulablepods.go:150, one call for the whole scan).  getPod is the pod lister's Get; rrPods
// the ResourceReservation cache as (namespace, appID) -> Status.Pods values; softPods the soft store as appID ->
// Reservations keys.  ok = false (no device, a record with an inexact quantity, any non-OK status): use the Go
// OverheadComputer.
func (o *OverheadRecords) OverheadForNodes(nodes []*v1.Node, getPod func(namespace, name string) (*v1.Pod, bool),
	rrPods map[[2]string][]string, softPods map[string][]string) (overhead, nonSchedulable resources.NodeGroupResources, warned int64, ok bool) {
	d, err := getDevice()
	if err != nil {
		return nil, nil, 0, false
	}
	o.mu.Lock()
	defer o.mu.Unlock()
	if o.nInexact > 0 {
		return nil, nil, 0, false
	}
	nodeIx := make(map[string]int32, len(o.nodeIx)+len(nodes)) // the record table's ids, plus listed nodes without records
	for k, v := range o.nodeIx {
		nodeIx[k] = v
	}
	query := make([]int32, len(nodes)+1)
	for i, n := range nodes {
		id, known := nodeIx[n.Name]
		if !known {
			id = int32(len(nodeIx))
			nodeIx[n.Name] = id
		}
		query[i] = id
	}
	keyIx, appIx, nameIx := map[[2]string]int32{}, map[string]int32{}, map[string]int32{}
	internName := func(s string) int32 {
		v, seen := nameIx[s]
		if !seen {
			v = int32(len(nameIx))
			nameIx[s] = v
		}
		return v
	}
	rrKey, rrName, rrOff := []int32{}, []int32{}, []int64{0}
	for k, names := range rrPods {
		keyIx[k] = int32(len(keyIx))
		rrKey = append(rrKey, keyIx[k])
		for _, s := range names {
			rrName = append(rrName, internName(s))
		}
		rrOff = append(rrOff, int64(len(rrName)))
	}
	softApp, softName, softOff := []int32{}, []int32{}, []int64{0}
	for app, names := range softPods {
		appIx[app] = int32(len(appIx))
		softApp = append(softApp, appIx[app])
		for _, s := range names {
			softName = append(softName, internName(s))
		}
		softOff = append(softOff, int64(len(softName)))
	}
	p := len(o.nodeID)
	listed, exe, spark := make([]uint8, p+1), make([]uint8, p+1), make([]uint8, p+1)
	ak, ai, nm := make([]int32, p+1), make([]int32, p+1), make([]int32, p+1)
	for i := 0; i < p; i++ {
		ak[i], ai[i] = -1, -1
		if o.nodeID[i] < 0 {
			continue
		}
		pod, found := getPod(o.ns[i], o.name[i])
		if !found {
			continue // overhead.go:131-138
		}
		listed[i] = 1
		if app, has := pod.Labels[common.SparkAppIDLabel]; has {
			k := [2]string{pod.Namespace, app}
			if _, seen := keyIx[k]; !seen {
				keyIx[k] = int32(len(keyIx))
			}
			if _, seen := appIx[app]; !seen {
				appIx[app] = int32(len(appIx))
			}
			ak[i], ai[i] = keyIx[k], appIx[app]
		}
		nm[i] = internName(pod.Name)
		if pod.Labels[common.SparkRoleLabel] == common.Executor {
			exe[i] = 1
		}
		if pod.Spec.SchedulerName == common.SparkSchedulerName {
			spark[i] = 1
		}
	}
	rrKey, rrName, softApp, softName = append(rrKey, 0), append(rrName, 0), append(softApp, 0), append(softName, 0) // non-empty bases
	nodeID := append(o.nodeID, -1)
	req := [3][]int64{append(o.req[0], 0), append(o.req[1], 0), append(o.req[2], 0)}
	n := len(nodes)
	outs := make([][]int64, 6)
	for k := range outs {
		outs[k] = make([]int64, n+1)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	d.mu.Lock()
	defer d.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, x := range []any{&nodeID[0], &listed[0], &exe[0], &spark[0], &ak[0], &ai[0], &nm[0], &query[0], &rrKey[0], &rrName[0],
		&rrOff[0], &softApp[0], &softName[0], &softOff[0], &req[0][0], &req[1][0], &req[2][0], &warned} {
		pin.Pin(x)
	}
	for k := range outs {
		pin.Pin(&outs[k][0])
	}
	pods := C.gp_overhead_pods{n_pods: C.int64_t(p), n_node_ids: C.int32_t(len(nodeIx)), n_app_keys: C.int32_t(len(keyIx)),
		n_app_ids: C.int32_t(len(appIx)), n_names: C.int32_t(len(nameIx)), node_id: ptr32(nodeID), req_cpu_milli: ptr64(req[0]),
		req_mem_bytes: ptr64(req[1]), req_gpu: ptr64(req[2]), listed: ptr8(listed), app_key: ptr32(ak), app_id: ptr32(ai),
		name_id: ptr32(nm), is_executor: ptr8(exe), spark_scheduler: ptr8(spark)}
	rsv := C.gp_overhead_reservations{n_rr: C.int32_t(len(rrOff) - 1), n_soft: C.int32_t(len(softOff) - 1),
		rr_app_key: ptr32(rrKey), rr_pod_off: ptr64(rrOff), rr_pod_name: ptr32(rrName),
		soft_app_id: ptr32(softApp), soft_pod_off: ptr64(softOff), soft_pod_name: ptr32(softName)}
	out := C.gp_overhead_out{overhead_cpu_milli: ptr64(outs[0]), overhead_mem_bytes: ptr64(outs[1]), overhead_gpu: ptr64(outs[2]),
		nonsched_cpu_milli: ptr64(outs[3]), nonsched_mem_bytes: ptr64(outs[4]), nonsched_gpu: ptr64(outs[5]),
		n_warned: (*C.int64_t)(unsafe.Pointer(&warned))}
	if C.gp_node_overhead(d.ctx, &pods, &rsv, C.int32_t(n), ptr32(query), &out) != C.GP_OK {
		return nil, nil, 0, false
	}
	overhead, nonSchedulable = resources.NodeGroupResources{}, resources.NodeGroupResources{}
	for i, node := range nodes {
		overhead[node.Name] = resources.CreateResources(outs[0][i], outs[1][i], outs[2][i])
		nonSchedulable[node.Name] = resources.CreateResources(outs[3][i], outs[4][i], outs[5][i])
	}
	return overhead, nonSchedulable, warned, true
}
