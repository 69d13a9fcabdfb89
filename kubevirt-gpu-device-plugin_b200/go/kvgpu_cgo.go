//go:build cgo

// Package device_plugin — cgo shim that routes the reference's discovery scan through libkvgpu.so.
//
// SOURCE ONLY: this image has no Go toolchain, so this file has never been compiled here (round-1 review
// findings — cgo pointer rule for the type dictionary, locking, range checks — are addressed in source).  It is
// the binding a maintainer of NVIDIA/kubevirt-gpu-device-plugin drops into pkg/device_plugin/
// next to device_plugin.go (see INTEGRATION.md).  It contains marshalling only — every decision
// (filter, join, bucketing, name sanitising) is made by the CUDA library behind include/kvgpu.h.
//
// It replaces the BODIES of three functions and keeps their signatures and side effects:
//
//	createIommuDeviceMap()            device_plugin.go:187  -> createIommuDeviceMapGPU()
//	createVgpuIDMap()                 device_plugin.go:255  -> createVgpuIDMapGPU()
//	getDeviceName(deviceID string)    device_plugin.go:371  -> getDeviceNameGPU(deviceID)
//
// The five sysfs readers stay the reference's own package variables (readIDFromFile, readLink,
// readNUMANode, readVgpuIDFromFile is replaced by a raw read, readGpuIDForVgpu :80-85), so the
// existing Ginkgo fakes keep working unchanged.
package device_plugin

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/.. -lkvgpu -Wl,-rpath,${SRCDIR}/..
#include <stdlib.h>
#include "kvgpu.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"io/fs"
	"log"
	"os"
	"path/filepath"
	"sort"
	"strconv"
	"strings"
	"sync"
	"unsafe"

	pluginapi "k8s.io/kubelet/pkg/apis/deviceplugin/v1beta1"
)

var kvgCtx *C.kvg_ctx
var kvgLoadedPath string

// A kvg_ctx is single-threaded (include/kvgpu.h).  The scans run on the main goroutine before any server
// starts, but getDeviceNameGPU, preferredAllocationGPU, allocateCheckGPU and the revalidate*GPU functions are reached from gRPC handler
// goroutines (grpc-go runs one goroutine per stream) and from healthCheck goroutines: every entry into the library
// takes kvgMu.
var kvgMu sync.Mutex

// kvgEnsure creates the context once and (re)loads the pci.ids table when the path changed.
// A CUDA failure is reported like the reference reports a failed walk: log + empty maps.
func kvgEnsure() error {
	if kvgCtx == nil {
		if rc := C.kvg_ctx_create(0, &kvgCtx); rc != C.KVG_OK {
			return fmt.Errorf("kvg_ctx_create: %d %s", int(rc), C.GoString(C.kvg_last_error(nil)))
		}
	}
	if kvgLoadedPath != pciIdsFilePath {
		data, err := os.ReadFile(pciIdsFilePath)
		if err != nil {
			log.Printf("Error opening pci ids file %s", pciIdsFilePath) // :375
			data = nil                                                  // empty table: every name is ""
		}
		var p *C.uint8_t
		if len(data) > 0 {
			p = (*C.uint8_t)(unsafe.Pointer(&data[0]))
		}
		if rc := C.kvg_pciids_load(kvgCtx, p, C.size_t(len(data))); rc != C.KVG_OK {
			return fmt.Errorf("kvg_pciids_load: %s", C.GoString(C.kvg_last_error(kvgCtx)))
		}
		kvgLoadedPath = pciIdsFilePath
	}
	return nil
}

func getDeviceNameGPU(deviceID string) string {
	kvgMu.Lock()
	defer kvgMu.Unlock()
	return getDeviceNameLocked(deviceID)
}

func getDeviceNameLocked(deviceID string) string {
	if err := kvgEnsure(); err != nil {
		log.Printf("Error: %v", err)
		return ""
	}
	out := make([]byte, 1<<17)
	var n C.size_t
	key := C.CString(deviceID)
	defer C.free(unsafe.Pointer(key))
	rc := C.kvg_name_lookup(kvgCtx, key, C.size_t(len(deviceID)), (*C.char)(unsafe.Pointer(&out[0])),
		C.size_t(len(out)), &n)
	if rc != C.KVG_OK {
		return ""
	}
	return string(out[:n])
}

func parseHex4(s string) (uint16, bool) {
	if len(s) != 4 {
		return 0, false
	}
	v, err := strconv.ParseUint(s, 16, 16)
	if err != nil || strings.ToLower(s) != s {
		return 0, false
	}
	return uint16(v), true
}

// createIommuDeviceMapGPU: same walk, same readers, same short-circuit order as :192-246, but the
// entries are only RECORDED (read failures become flag bits); the GPU filters, joins and buckets.
func createIommuDeviceMapGPU() {
	kvgMu.Lock()
	defer kvgMu.Unlock()
	iommuMap = make(map[string][]NvidiaGpuDevice)
	deviceMap = make(map[string][]NvidiaGpuDevice)
	bdfToIommuMap = make(map[string]string)
	var names []string
	var recs []C.kvg_pci_rec
	groupIDs := map[string]uint32{}
	var groupNames []string
	// `device` strings travel in index mode: the reference keeps WHATEVER the file holds as the map key
	// (:240, :294-302), so the record carries an interned id and the string stays here
	deviceIDs := map[string]uint16{}
	var deviceNames []string
	rangeErr := ""
	filepath.Walk(basePath, func(path string, info os.FileInfo, err error) error {
		if err != nil {
			log.Printf("Error accessing file path %q: %v\n", path, err)
			return err
		}
		if info.IsDir() {
			return nil
		}
		var r C.kvg_pci_rec
		r.addr = C.uint32_t(len(names)) // index mode: names[] maps the handle back
		r.vendor = 0xffff
		vendorID, err := readIDFromFile(basePath, info.Name(), "vendor")
		if err != nil {
			r.flags |= C.KVG_PF_VENDOR_ERR
		} else if v, ok := parseHex4(vendorID); ok {
			r.vendor = C.uint16_t(v)
		}
		if err == nil && vendorID == nvidiaVendorID {
			driver, err := readLink(basePath, info.Name(), "driver")
			switch {
			case err != nil:
				r.flags |= C.KVG_PF_DRIVER_ERR
			case driver == "vfio-pci":
				r.driver = C.KVG_DRV_VFIO_PCI
			case driver == "nvgrace_gpu_vfio_pci":
				r.driver = C.KVG_DRV_NVGRACE
			default:
				r.driver = C.KVG_DRV_OTHER
			}
			if err == nil && isSupportedVfioDriver(driver) {
				iommuGroup, err := readLink(basePath, info.Name(), "iommu_group")
				if err != nil {
					r.flags |= C.KVG_PF_IOMMU_ERR
				} else {
					id, ok := groupIDs[iommuGroup]
					if !ok {
						id = uint32(len(groupNames))
						groupIDs[iommuGroup] = id
						groupNames = append(groupNames, iommuGroup)
					}
					r.iommu_group = C.uint32_t(id)
					numaNode, err := readNUMANode(basePath, info.Name())
					if err != nil {
						r.flags |= C.KVG_PF_NUMA_ERR
					} else if numaNode < -32768 || numaNode > 32767 {
						// the 16-byte record carries an int16: refuse loudly (kvgpu/plugin.py: KVG_ERANGE)
						rangeErr = fmt.Sprintf("numa_node %d of %s does not fit the wire format", numaNode, info.Name())
					}
					r.numa = C.int16_t(numaNode)
					deviceID, err := readIDFromFile(basePath, info.Name(), "device")
					if err != nil {
						r.flags |= C.KVG_PF_DEVICE_ERR
					} else {
						id, ok := deviceIDs[deviceID]
						if !ok {
							if len(deviceNames) > 0xffff {
								rangeErr = "more than 65536 distinct device strings"
							}
							id = uint16(len(deviceNames))
							deviceIDs[deviceID] = id
							deviceNames = append(deviceNames, deviceID)
						}
						r.device = C.uint16_t(id)
					}
				}
			}
		}
		names = append(names, info.Name())
		recs = append(recs, r)
		return nil
	})
	if rangeErr != "" {
		log.Printf("Error: %s", rangeErr) // maps stay empty, like a failed walk (:193-196)
		return
	}
	if err := kvgEnsure(); err != nil {
		log.Printf("Error: %v", err) // maps stay empty, like a failed walk (:193-196)
		return
	}
	var res *C.kvg_pci_result
	var p *C.kvg_pci_rec
	if len(recs) > 0 {
		p = &recs[0]
	}
	if rc := C.kvg_scan_pci(kvgCtx, p, C.size_t(len(recs)), &res); rc != C.KVG_OK {
		log.Printf("Error: kvg_scan_pci: %s", C.GoString(C.kvg_last_error(kvgCtx)))
		return
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	S := int(res.n_survivors)
	surv := unsafe.Slice(res.survivors, S)
	dev := func(i uint32) NvidiaGpuDevice {
		return NvidiaGpuDevice{addr: names[surv[i].addr], numaNode: int64(surv[i].numa)}
	}
	devKeys := unsafe.Slice(res.dev_keys, int(res.n_dev_keys))
	devOff := unsafe.Slice(res.dev_off, int(res.n_dev_keys)+1)
	devPerm := unsafe.Slice(res.dev_perm, S)
	for k := range devKeys {
		key := deviceNames[devKeys[k]] // index mode; getDeviceName(key) is asked later with these exact bytes
		for _, i := range devPerm[devOff[k]:devOff[k+1]] {
			deviceMap[key] = append(deviceMap[key], dev(uint32(i)))
		}
	}
	grpKeys := unsafe.Slice(res.grp_keys, int(res.n_groups))
	grpOff := unsafe.Slice(res.grp_off, int(res.n_groups)+1)
	grpPerm := unsafe.Slice(res.grp_perm, S)
	for k := range grpKeys {
		g := groupNames[grpKeys[k]]
		for _, i := range grpPerm[grpOff[k]:grpOff[k+1]] {
			iommuMap[g] = append(iommuMap[g], dev(uint32(i)))
		}
	}
	for i := 0; i < S; i++ {
		bdfToIommuMap[names[surv[i].addr]] = groupNames[surv[i].iommu_group]
	}
}

// createIommuDeviceMapRawGPU: createIommuDeviceMap (:187-247) with every reader's rule on the GPU.  The walk makes the
// five reads of every entry and decodes nothing; kvg_scan_pci_raw applies readIDFromFileFunc, readLinkFunc,
// readNUMANodeFunc and isSupportedVfioDriver in the reference's order, chooses the snapshot modes and scans.
func createIommuDeviceMapRawGPU() {
	kvgMu.Lock()
	defer kvgMu.Unlock()
	iommuMap = make(map[string][]NvidiaGpuDevice)
	deviceMap = make(map[string][]NvidiaGpuDevice)
	bdfToIommuMap = make(map[string]string)
	var names []string
	var bytes []byte
	off := []uint32{0}
	var state []uint16
	filepath.Walk(basePath, func(path string, info os.FileInfo, err error) error {
		if err != nil {
			log.Printf("Error accessing file path %q: %v\n", path, err)
			return err
		}
		if info.IsDir() {
			return nil
		}
		name := info.Name()
		var st uint16
		bytes = append(bytes, name...)
		off = append(off, uint32(len(bytes)))
		for f, prop := range []string{"vendor", "driver", "iommu_group", "numa_node", "device"} {
			p := filepath.Join(basePath, name, prop)
			var data []byte
			var err error
			if prop == "driver" || prop == "iommu_group" {
				var t string
				t, err = os.Readlink(p)
				data = []byte(t)
			} else {
				data, err = os.ReadFile(p)
			}
			st |= 1 << (f + 1)
			if err != nil {
				st |= 1 << (8 + f + 1)
				data = nil
			}
			bytes = append(bytes, data...)
			off = append(off, uint32(len(bytes)))
		}
		names = append(names, name)
		state = append(state, st)
		return nil
	})
	if err := kvgEnsure(); err != nil {
		log.Printf("Error: %v", err) // maps stay empty, like a failed walk (:193-196)
		return
	}
	// the library copies the inputs before it returns (cgo pointer rule): C copies of them
	var raw C.kvg_pci_raw
	raw.n = C.size_t(len(state))
	if len(state) > 0 {
		raw.off = (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&off[0])), 4*len(off))))
		raw.state = (*C.uint16_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&state[0])), 2*len(state))))
		raw.bytes = (*C.uint8_t)(C.CBytes(append(bytes, 0)))
		defer C.free(unsafe.Pointer(raw.off))
		defer C.free(unsafe.Pointer(raw.state))
		defer C.free(unsafe.Pointer(raw.bytes))
	}
	var res *C.kvg_pci_result
	var snap *C.kvg_pci_snap
	if rc := C.kvg_scan_pci_raw(kvgCtx, &raw, &res, &snap); rc != C.KVG_OK {
		// KVG_EPANIC: the reference would panic here; the maps stay empty
		log.Printf("Error: kvg_scan_pci_raw: %s", C.GoString(C.kvg_last_error(kvgCtx)))
		return
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	defer C.kvg_result_free(unsafe.Pointer(snap))
	table := func(n C.uint32_t, o *C.uint32_t, b *C.uint8_t) []string {
		if n == 0 {
			return nil
		}
		offs := unsafe.Slice(o, int(n)+1)
		all := C.GoBytes(unsafe.Pointer(b), C.int(offs[n]))
		out := make([]string, int(n))
		for h := range out {
			out[h] = string(all[offs[h]:offs[h+1]])
		}
		return out
	}
	groupNames := table(snap.n_group_names, snap.group_off, snap.group_bytes)
	deviceNames := table(snap.n_device_names, snap.device_off, snap.device_bytes)
	S := int(res.n_survivors)
	surv := unsafe.Slice(res.survivors, S)
	addr := func(i uint32) string {
		a := uint32(surv[i].addr)
		if snap.packed_addr == 0 {
			return names[a]
		}
		return fmt.Sprintf("%04x:%02x:%02x.%x", a>>16, (a>>8)&0xff, (a>>3)&0x1f, a&7)
	}
	group := func(g C.uint32_t) string {
		if snap.groups_numeric != 0 {
			return strconv.FormatUint(uint64(g), 10)
		}
		return groupNames[g]
	}
	dev := func(i uint32) NvidiaGpuDevice { return NvidiaGpuDevice{addr: addr(i), numaNode: int64(surv[i].numa)} }
	devKeys := unsafe.Slice(res.dev_keys, int(res.n_dev_keys))
	devOff := unsafe.Slice(res.dev_off, int(res.n_dev_keys)+1)
	devPerm := unsafe.Slice(res.dev_perm, S)
	for k := range devKeys {
		key := fmt.Sprintf("%04x", uint16(devKeys[k]))
		if snap.devices_numeric == 0 {
			key = deviceNames[devKeys[k]] // getDeviceName(key) is asked later with these exact bytes
		}
		for _, i := range devPerm[devOff[k]:devOff[k+1]] {
			deviceMap[key] = append(deviceMap[key], dev(uint32(i)))
		}
	}
	grpKeys := unsafe.Slice(res.grp_keys, int(res.n_groups))
	grpOff := unsafe.Slice(res.grp_off, int(res.n_groups)+1)
	grpPerm := unsafe.Slice(res.grp_perm, S)
	for k := range grpKeys {
		g := group(grpKeys[k])
		for _, i := range grpPerm[grpOff[k]:grpOff[k+1]] {
			iommuMap[g] = append(iommuMap[g], dev(uint32(i)))
		}
	}
	for i := 0; i < S; i++ {
		bdfToIommuMap[addr(uint32(i))] = group(surv[i].iommu_group)
	}
}

// createVgpuIDMapGPU: :259-290 with the label rule (:341-342) and both group-bys on the GPU.
func createVgpuIDMapGPU() {
	kvgMu.Lock()
	defer kvgMu.Unlock()
	vGpuMap = make(map[string][]NvidiaGpuDevice)
	gpuVgpuMap = make(map[string][]string)
	var names, parentNames []string
	var recs []C.kvg_mdev_rec
	typeIDs := map[string]uint16{}
	var rawTypes [][]byte
	parentIDs := map[string]uint32{}
	filepath.Walk(vGpuBasePath, func(path string, info os.FileInfo, err error) error {
		if err != nil {
			return err
		}
		if info.IsDir() {
			return nil
		}
		var r C.kvg_mdev_rec
		idx := uint32(len(names))
		r.uuid[0], r.uuid[1], r.uuid[2], r.uuid[3] = C.uint8_t(idx>>24), C.uint8_t(idx>>16), C.uint8_t(idx>>8), C.uint8_t(idx)
		raw, err := os.ReadFile(filepath.Join(vGpuBasePath, info.Name(), "mdev_type/name")) // raw: the GPU sanitises
		if err != nil {
			r.flags |= C.KVG_MF_TYPE_ERR
		} else {
			id, ok := typeIDs[string(raw)]
			if !ok {
				id = uint16(len(rawTypes))
				typeIDs[string(raw)] = id
				rawTypes = append(rawTypes, raw)
			}
			r.type_idx = C.uint16_t(id)
			gpuID, err := readGpuIDForVgpu(vGpuBasePath, info.Name())
			if err != nil {
				r.flags |= C.KVG_MF_PARENT_ERR
			} else {
				id, ok := parentIDs[gpuID]
				if !ok {
					id = uint32(len(parentNames))
					parentIDs[gpuID] = id
					parentNames = append(parentNames, gpuID)
				}
				r.parent = C.uint32_t(id)
				numaNode, err := readNUMANode(basePath, gpuID)
				if err != nil {
					r.flags |= C.KVG_MF_NUMA_ERR
				}
				r.parent_numa = C.int16_t(numaNode)
			}
		}
		names = append(names, info.Name())
		recs = append(recs, r)
		return nil
	})
	if err := kvgEnsure(); err != nil {
		log.Printf("Error: %v", err)
		return
	}
	dict, freeDict := cTypeDict(rawTypes)
	defer freeDict()
	var res *C.kvg_mdev_result
	var p *C.kvg_mdev_rec
	if len(recs) > 0 {
		p = &recs[0]
	}
	if rc := C.kvg_scan_mdev(kvgCtx, p, C.size_t(len(recs)), &dict, &res); rc != C.KVG_OK {
		log.Printf("Error: kvg_scan_mdev: %s", C.GoString(C.kvg_last_error(kvgCtx)))
		return
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	S := int(res.n_survivors)
	surv := unsafe.Slice(res.survivors, S)
	labelOff := unsafe.Slice(res.label_off, int(res.n_types)+1)
	labels := unsafe.Slice((*byte)(unsafe.Pointer(res.label_bytes)), int(labelOff[res.n_types]))
	tKeys := unsafe.Slice(res.type_keys, int(res.n_type_keys))
	tOff := unsafe.Slice(res.type_off, int(res.n_type_keys)+1)
	tPerm := unsafe.Slice(res.type_perm, S)
	for k := range tKeys {
		t := tKeys[k]
		label := string(labels[labelOff[t]:labelOff[t+1]])
		for _, i := range tPerm[tOff[k]:tOff[k+1]] {
			vGpuMap[label] = append(vGpuMap[label], NvidiaGpuDevice{addr: names[surv[i].src], numaNode: int64(surv[i].numa)})
		}
	}
	pKeys := unsafe.Slice(res.par_keys, int(res.n_parents))
	pOff := unsafe.Slice(res.par_off, int(res.n_parents)+1)
	pPerm := unsafe.Slice(res.par_perm, S)
	for k := range pKeys {
		g := parentNames[pKeys[k]]
		for _, i := range pPerm[pOff[k]:pOff[k+1]] {
			gpuVgpuMap[g] = append(gpuVgpuMap[g], names[surv[i].src])
		}
	}
	_ = sort.Strings // (kept: callers that want deterministic logs sort the keys)
}

// createVgpuIDMapRawGPU: createVgpuIDMap (:255-291) with every reader's rule on the GPU.  The walk reads the type file,
// the entry's link target and the parent's numa_node and decodes nothing; kvg_scan_mdev_raw applies
// readGpuIDForVgpuFunc, readNUMANodeFunc, the type dictionary and the snapshot modes, then scans.  The one thing
// derived here is the numa_node path, which needs the parent component of the target (strings.Split(t, "/")[len-2],
// Trim "\n"); the GPU decodes the parent key itself.  A vGPU with an empty parent is listed under gpuVgpuMap[""], as
// in the reference.  Source only, like the rest of this file: it has never been compiled.
func createVgpuIDMapRawGPU() {
	kvgMu.Lock()
	defer kvgMu.Unlock()
	vGpuMap = make(map[string][]NvidiaGpuDevice)
	gpuVgpuMap = make(map[string][]string)
	var names []string
	var bytes []byte
	off := []uint32{0}
	var state []uint16
	filepath.Walk(vGpuBasePath, func(path string, info os.FileInfo, err error) error {
		if err != nil {
			return err
		}
		if info.IsDir() {
			return nil
		}
		name := info.Name()
		var st uint16
		field := func(f int, data []byte, err error) {
			st |= 1 << f
			if err != nil {
				st |= 1 << (8 + f)
				data = nil
			}
			bytes = append(bytes, data...)
			off = append(off, uint32(len(bytes)))
		}
		bytes = append(bytes, name...)
		off = append(off, uint32(len(bytes)))
		data, err := os.ReadFile(filepath.Join(vGpuBasePath, name, "mdev_type/name"))
		field(C.KVG_MRAW_TYPE, data, err)
		target, lerr := os.Readlink(filepath.Join(vGpuBasePath, name))
		field(C.KVG_MRAW_LINK, []byte(target), lerr)
		parts := strings.Split(target, "/")
		if lerr == nil && len(parts) >= 2 {
			data, err = os.ReadFile(filepath.Join(basePath, strings.Trim(parts[len(parts)-2], "\n"), "numa_node"))
			field(C.KVG_MRAW_NUMA, data, err)
		} else {
			off = append(off, uint32(len(bytes))) // not reached by the reference: not made
		}
		names = append(names, name)
		state = append(state, st)
		return nil
	})
	if err := kvgEnsure(); err != nil {
		log.Printf("Error: %v", err)
		return
	}
	var raw C.kvg_mdev_raw
	raw.n = C.size_t(len(state))
	if len(state) > 0 {
		raw.off = (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&off[0])), 4*len(off))))
		raw.state = (*C.uint16_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&state[0])), 2*len(state))))
		raw.bytes = (*C.uint8_t)(C.CBytes(append(bytes, 0)))
		defer C.free(unsafe.Pointer(raw.off))
		defer C.free(unsafe.Pointer(raw.state))
		defer C.free(unsafe.Pointer(raw.bytes))
	}
	var res *C.kvg_mdev_result
	var snap *C.kvg_mdev_snap
	if rc := C.kvg_scan_mdev_raw(kvgCtx, &raw, &res, &snap); rc != C.KVG_OK {
		// KVG_EPANIC: the reference would panic here; the maps stay empty
		log.Printf("Error: kvg_scan_mdev_raw: %s", C.GoString(C.kvg_last_error(kvgCtx)))
		return
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	defer C.kvg_result_free(unsafe.Pointer(snap))
	var parentNames []string
	if snap.parents_packed == 0 && snap.n_parent_names > 0 {
		offs := unsafe.Slice(snap.parent_off, int(snap.n_parent_names)+1)
		all := C.GoBytes(unsafe.Pointer(snap.parent_bytes), C.int(offs[snap.n_parent_names]))
		for h := 0; h < int(snap.n_parent_names); h++ {
			parentNames = append(parentNames, string(all[offs[h]:offs[h+1]]))
		}
	}
	S := int(res.n_survivors)
	surv := unsafe.Slice(res.survivors, S)
	uuid := func(i uint32) string {
		if snap.uuid_ok == 0 {
			return names[surv[i].src]
		}
		u := surv[i].uuid
		return fmt.Sprintf("%x-%x-%x-%x-%x", u[0:4], u[4:6], u[6:8], u[8:10], u[10:16])
	}
	parent := func(p C.uint32_t) string {
		if snap.parents_packed == 0 {
			return parentNames[p]
		}
		a := uint32(p)
		return fmt.Sprintf("%04x:%02x:%02x.%x", a>>16, (a>>8)&0xff, (a>>3)&0x1f, a&7)
	}
	labelOff := unsafe.Slice(res.label_off, int(res.n_types)+1)
	labels := unsafe.Slice((*byte)(unsafe.Pointer(res.label_bytes)), int(labelOff[res.n_types]))
	tKeys := unsafe.Slice(res.type_keys, int(res.n_type_keys))
	tOff := unsafe.Slice(res.type_off, int(res.n_type_keys)+1)
	tPerm := unsafe.Slice(res.type_perm, S)
	for k := range tKeys {
		t := tKeys[k]
		label := string(labels[labelOff[t]:labelOff[t+1]])
		for _, i := range tPerm[tOff[k]:tOff[k+1]] {
			vGpuMap[label] = append(vGpuMap[label], NvidiaGpuDevice{addr: uuid(uint32(i)), numaNode: int64(surv[i].numa)})
		}
	}
	pKeys := unsafe.Slice(res.par_keys, int(res.n_parents))
	pOff := unsafe.Slice(res.par_off, int(res.n_parents)+1)
	pPerm := unsafe.Slice(res.par_perm, S)
	for k := range pKeys {
		g := parent(pKeys[k])
		for _, i := range pPerm[pOff[k]:pOff[k+1]] {
			gpuVgpuMap[g] = append(gpuVgpuMap[g], uuid(uint32(i)))
		}
	}
}

// cTypeDict lays raw out as a kvg_type_dict.  The dictionary struct holds two pointers: they must not be Go pointers
// (cgo rule: a Go pointer passed to C may not point at memory that itself holds Go pointers), so both arrays live in
// C memory; free releases them after the call.
func cTypeDict(raw [][]byte) (dict C.kvg_type_dict, free func()) {
	total := 0
	for _, t := range raw {
		total += len(t)
	}
	cOff := (*C.uint32_t)(C.malloc(C.size_t(4 * (len(raw) + 1))))
	cBlob := (*C.uint8_t)(C.malloc(C.size_t(total + 1)))
	off := unsafe.Slice(cOff, len(raw)+1)
	blob := unsafe.Slice((*byte)(unsafe.Pointer(cBlob)), total+1)
	off[0] = 0
	pos := 0
	for i, t := range raw {
		pos += copy(blob[pos:], t)
		off[i+1] = C.uint32_t(pos)
	}
	blob[total] = 0
	return C.kvg_type_dict{n_types: C.uint32_t(len(raw)), off: cOff, bytes: cBlob}, func() {
		C.free(unsafe.Pointer(cOff))
		C.free(unsafe.Pointer(cBlob))
	}
}

// revalidateBatchGPU is the Allocate-time re-check of generic_device_plugin.go:387-399 for ALL devices
// of a container request in one pass of the classification kernel (Python twin:
// kvgpu/serve.py BatchRevalidator, pinned by tests/test_serve.py).  devs[i] is re-read with the
// reference's own readers, in the reference's order; want[i] is the IOMMU group the maps hold for it.
// It returns the index of the first device the reference would reject, or -1.
//
// The record's driver is pinned to vfio-pci and its device id to 0 because Allocate re-checks only the
// group link and the vendor; K3's predicate is then exactly "vendor is 10de and both reads worked" and
// the survivor's interned group id says whether the link still points at the expected group.
//
// Call site (generic_device_plugin.go:376-416): collect (dev.addr, iommuId) for every dev of every
// requested BDF, call this once, and return the "unknown device" error for devs[first] if first >= 0.
func revalidateBatchGPU(devs []string, want []string) (first int, err error) {
	if len(devs) == 0 {
		return -1, nil
	}
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return 0, err
	}
	intern := map[string]uint32{}
	id := func(s string) uint32 {
		if v, ok := intern[s]; ok {
			return v
		}
		v := uint32(len(intern))
		intern[s] = v
		return v
	}
	recs := make([]C.kvg_pci_rec, len(devs))
	for i, addr := range devs {
		r := &recs[i]
		r.addr = C.uint32_t(i)
		r.vendor = 0xffff
		r.driver = C.KVG_DRV_VFIO_PCI
		r.iommu_group = C.uint32_t(id(want[i]))
		group, err := readLink(basePath, addr, "iommu_group")
		if err != nil {
			r.flags |= C.KVG_PF_IOMMU_ERR
		} else {
			r.iommu_group = C.uint32_t(id(group))
		}
		vendorID, err := readIDFromFile(basePath, addr, "vendor")
		if err != nil {
			r.flags |= C.KVG_PF_VENDOR_ERR
		} else if vendorID == nvidiaVendorID {
			r.vendor = 0x10de
		}
	}
	var res *C.kvg_pci_result
	if rc := C.kvg_scan_pci(kvgCtx, &recs[0], C.size_t(len(recs)), &res); rc != C.KVG_OK {
		return 0, fmt.Errorf("kvg_scan_pci: %s", C.GoString(C.kvg_last_error(kvgCtx)))
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	ok := make(map[uint32]uint32, int(res.n_survivors))
	for _, s := range unsafe.Slice(res.survivors, int(res.n_survivors)) {
		ok[uint32(s.addr)] = uint32(s.iommu_group)
	}
	for i := range devs {
		if g, alive := ok[uint32(i)]; !alive || g != intern[want[i]] {
			return i, nil
		}
	}
	return -1, nil
}

// revalidateGroupsGPU is the same re-check as revalidateBatchGPU, with the same contract and call site, as its own
// rule in one launch of kvg_pci_group_check (Python twin: kvgpu/serve.py GroupCheck, tested against BatchRevalidator
// by tests/test_serve_group_check.py).  A device passes iff its iommu_group link read back as want[i] and its vendor
// as "10de" (generic_device_plugin.go:388-397); no driver or device id is pinned, because the rule reads neither.
// The group strings are interned per call and never parsed as numbers: the reference compares strings, so "042" is
// not "42".  It touches no scan state, so it may run while a scan's result is still to be fetched.
func revalidateGroupsGPU(devs []string, want []string) (first int, err error) {
	if len(devs) == 0 {
		return -1, nil
	}
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return 0, err
	}
	intern := map[string]uint32{}
	id := func(s string) uint32 {
		if v, ok := intern[s]; ok {
			return v
		}
		v := uint32(len(intern))
		intern[s] = v
		return v
	}
	recs := make([]C.kvg_pci_rec, len(devs))
	wantGroup := make([]C.uint32_t, len(devs))
	for i, addr := range devs {
		r := &recs[i]
		r.addr = C.uint32_t(i)
		r.vendor = 0xffff
		wantGroup[i] = C.uint32_t(id(want[i]))
		group, err := readLink(basePath, addr, "iommu_group")
		if err != nil {
			r.flags |= C.KVG_PF_IOMMU_ERR
		} else {
			r.iommu_group = C.uint32_t(id(group))
		}
		vendorID, err := readIDFromFile(basePath, addr, "vendor")
		if err != nil {
			r.flags |= C.KVG_PF_VENDOR_ERR
		} else if vendorID == nvidiaVendorID {
			r.vendor = 0x10de
		}
	}
	var bad C.size_t
	if rc := C.kvg_pci_group_check(kvgCtx, &recs[0], &wantGroup[0], C.size_t(len(recs)), &bad); rc != C.KVG_OK {
		return 0, fmt.Errorf("kvg_pci_group_check: %s", C.GoString(C.kvg_last_error(kvgCtx)))
	}
	if int(bad) == len(devs) {
		return -1, nil
	}
	return int(bad), nil
}

// allocMember is one member of a requested IOMMU group, as Allocate visits it: its address and the group the maps
// hold for it.
type allocMember struct{ addr, group string }

// allocDecision is what allocateCheckGPU decides for one container request.
type allocDecision struct {
	bad   int         // position of the first member the reference rejects, or -1
	panic interface{} // what that member's vendor read panicked with, when the reference reaches the read; else nil
	egm   []string    // the EGM device paths to mount, sorted (egmPathsForAllocatedGPUs :159-184)
}

// allocateCheckGPU takes every decision of the passthrough plugin's Allocate (generic_device_plugin.go:352-444) for
// all container requests of one AllocateRequest in one launch of kvg_pci_allocate_check (Python twin: kvgpu/serve.py
// AllocateCheck, tested against GroupCheck and the CPU EGM rule by tests/test_serve_allocate_check.py).  It is the
// twin of revalidateGroupsGPU and egmPathsForAllocatedGPUs together: members[r] lists request r's group members in
// the reference's order, ids[r] its DevicesIDs.  Every member's link and vendor are read with the reference's
// readers, request by request; a panicking read is recovered per member and handed back only when the reference
// would reach it.  The EGM strings are interned with the reference's own strings.ToLower(strings.TrimSpace(s)), so
// the keys are exactly the ones egmPathsForAllocatedGPUs compares.  The caller replays each request in the
// reference's order (lookup error, re-check failure or panic, iommufd read, requested device found, EGM specs) and
// returns the first error of the first failing request.  It touches no scan state.
func allocateCheckGPU(members [][]allocMember, ids [][]string, egmDevices []EGMDeviceInfo) ([]allocDecision, error) {
	if len(members) == 0 {
		return nil, nil
	}
	key := func(s string) string { return strings.ToLower(strings.TrimSpace(s)) }
	egmHandle := map[string]uint32{}
	egmOff, egmGPU := []C.uint32_t{}, []C.uint32_t{}
	if len(egmDevices) > 0 {
		egmOff = append(egmOff, 0)
	}
	for _, e := range egmDevices {
		for _, g := range e.GPUBDFs {
			h, ok := egmHandle[key(g)]
			if !ok {
				h = uint32(len(egmHandle))
				egmHandle[key(g)] = h
			}
			egmGPU = append(egmGPU, C.uint32_t(h))
		}
		egmOff = append(egmOff, C.uint32_t(len(egmGPU)))
	}
	nEgmGPUs := uint32(len(egmHandle))
	intern := map[string]uint32{}
	id := func(s string) uint32 {
		if v, ok := intern[s]; ok {
			return v
		}
		v := uint32(len(intern))
		intern[s] = v
		return v
	}
	creqs := make([]C.kvg_alloc_req, len(members))
	recs, wantGroup, cids := []C.kvg_pci_rec{}, []C.uint32_t{}, []C.uint32_t{}
	linkOK, panics := []bool{}, map[int]interface{}{}
	for r, ms := range members {
		for _, m := range ms {
			i := len(recs)
			rec := C.kvg_pci_rec{addr: C.uint32_t(i), vendor: 0xffff}
			wantGroup = append(wantGroup, C.uint32_t(id(m.group)))
			group, err := readLink(basePath, m.addr, "iommu_group")
			ok := false
			if err != nil {
				rec.flags |= C.KVG_PF_IOMMU_ERR
			} else {
				rec.iommu_group = C.uint32_t(id(group))
				ok = group == m.group
			}
			vendorID, err := func() (v string, err error) {
				defer func() {
					if p := recover(); p != nil {
						panics[i], err = p, fmt.Errorf("panic")
					}
				}()
				return readIDFromFile(basePath, m.addr, "vendor")
			}()
			if err != nil {
				rec.flags |= C.KVG_PF_VENDOR_ERR
			} else if vendorID == nvidiaVendorID {
				rec.vendor = 0x10de
			}
			recs = append(recs, rec)
			linkOK = append(linkOK, ok)
		}
		for _, d := range ids[r] {
			h, ok := egmHandle[key(d)]
			if !ok {
				h = nEgmGPUs
			}
			cids = append(cids, C.uint32_t(h))
		}
		creqs[r] = C.kvg_alloc_req{n_members: C.uint32_t(len(ms)), n_ids: C.uint32_t(len(ids[r]))}
	}
	firstBad := make([]C.uint32_t, len(members))
	take := make([]C.uint8_t, len(members)*len(egmDevices)+1)
	var recp *C.kvg_pci_rec
	var wantp, idp, offp, gpup *C.uint32_t
	if len(recs) > 0 {
		recp, wantp = &recs[0], &wantGroup[0]
	}
	if len(cids) > 0 {
		idp = &cids[0]
	}
	if len(egmOff) > 0 {
		offp = &egmOff[0]
	}
	if len(egmGPU) > 0 {
		gpup = &egmGPU[0]
	}
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return nil, err
	}
	if rc := C.kvg_pci_allocate_check(kvgCtx, &creqs[0], C.uint32_t(len(creqs)), recp, wantp, C.size_t(len(recs)), idp,
		C.size_t(len(cids)), offp, gpup, C.uint32_t(len(egmDevices)), C.uint32_t(nEgmGPUs), &firstBad[0],
		&take[0]); rc != C.KVG_OK {
		return nil, fmt.Errorf("kvg_pci_allocate_check: %s", C.GoString(C.kvg_last_error(kvgCtx)))
	}
	out := make([]allocDecision, len(members))
	at := 0
	for r, ms := range members {
		d := allocDecision{bad: -1, egm: []string{}}
		if b := int(firstBad[r]); b < len(ms) {
			d.bad = b
			if linkOK[at+b] {
				d.panic = panics[at+b]
			}
		}
		for e, dev := range egmDevices {
			if take[r*len(egmDevices)+e] != 0 {
				d.egm = append(d.egm, dev.DevPath)
			}
		}
		sort.Strings(d.egm)
		out[r] = d
		at += len(ms)
	}
	return out, nil
}

// preferredAllocationGPU is GetPreferredAllocation's NUMA packing (generic_device_plugin.go:470-608) for every container
// request of one PreferredAllocationRequest, in one launch of kvg_preferred_allocation (Python twin: kvgpu/serve.py
// NumaPacker, tested against serve.preferred_allocation by tests/test_serve_preferred_alloc.py).  devs is the plugin's
// device list: the last entry with topology gives a device its node, and a node of -1, a device without topology and
// an ID the plugin does not know share the reference's -1 group (KVG_PREF_NODE_NONE).  Per request the ID strings,
// must-include first, are interned into handles and the node values into dense indices; the kernel decides, and this
// function only maps the positions it returns back to IDs.  The error is the reference's text for the first failing
// request.  It touches no scan state, so it may run while a scan's result is still to be fetched.
func preferredAllocationGPU(devs []*pluginapi.Device, reqs []*pluginapi.ContainerPreferredAllocationRequest) ([][]string, error) {
	if len(reqs) == 0 {
		return nil, nil
	}
	nodeOf := map[string]int64{}
	for _, d := range devs {
		if d.Topology != nil && len(d.Topology.Nodes) > 0 {
			nodeOf[d.ID] = d.Topology.Nodes[0].ID
		}
	}
	creqs := make([]C.kvg_pref_req, len(reqs))
	ids := []C.kvg_pref_id{}
	entries := make([][]string, len(reqs))
	for r, req := range reqs {
		ent := append(append([]string{}, req.MustIncludeDeviceIDs...), req.AvailableDeviceIDs...)
		handles, nodes := map[string]uint32{}, map[int64]uint32{}
		for _, id := range ent {
			h, ok := handles[id]
			if !ok {
				h = uint32(len(handles))
				handles[id] = h
			}
			node := uint32(C.KVG_PREF_NODE_NONE)
			if n, ok := nodeOf[id]; ok && n != -1 {
				v, ok := nodes[n]
				if !ok {
					v = uint32(len(nodes))
					nodes[n] = v
				}
				node = v
			}
			ids = append(ids, C.kvg_pref_id{handle: C.uint32_t(h), node: C.uint32_t(node)})
		}
		creqs[r] = C.kvg_pref_req{n_must: C.uint32_t(len(req.MustIncludeDeviceIDs)),
			n_avail: C.uint32_t(len(req.AvailableDeviceIDs)), size: C.int32_t(req.AllocationSize)}
		entries[r] = ent
	}
	res := make([]C.kvg_pref_res, len(reqs))
	pos := make([]C.uint32_t, len(ids)+1)
	var idp *C.kvg_pref_id
	if len(ids) > 0 {
		idp = &ids[0]
	}
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return nil, err
	}
	if rc := C.kvg_preferred_allocation(kvgCtx, &creqs[0], C.uint32_t(len(creqs)), idp, C.size_t(len(ids)), &res[0],
		&pos[0]); rc != C.KVG_OK {
		return nil, fmt.Errorf("kvg_preferred_allocation: %s", C.GoString(C.kvg_last_error(kvgCtx)))
	}
	out := make([][]string, len(reqs))
	at := 0
	for r, ent := range entries {
		if res[r].n_out < 0 {
			return nil, fmt.Errorf("number of MustIncludeDeviceIDs (%d) exceeds allocation size (%d)",
				int(res[r].n_must_distinct), reqs[r].AllocationSize)
		}
		out[r] = make([]string, int(res[r].n_out))
		for k := range out[r] {
			out[r][k] = ent[pos[at+k]]
		}
		at += len(ent)
	}
	return out, nil
}

// revalidateVgpuBatchGPU is the Allocate-time re-check of generic_vgpu_device_plugin.go:216-228 for ALL IDs of an
// AllocateRequest in one launch (Python twin: kvgpu/serve.py MdevLabelCheck, pinned by
// tests/test_serve_vgpu_allocate.py).  Each ID's mdev_type/name is read raw, as readVgpuIDFromFile reads it, and no
// regexp runs here: the GPU applies Trim(raw, "\n") and \s+ -> "_" (device_plugin.go:341-342) and compares the label
// with deviceName.  keep[i] is false for an ID whose read failed; such a file never reaches the rule.
//
// Call site (generic_vgpu_device_plugin.go:208-245): collect the DevicesIDs of every ContainerRequest in order, call
// this once, then walk the requests again and append each devID whose keep entry is true to that container's env
// list, replacing the per-ID readVgpuIDFromFile call and its regexp.MustCompile.
func revalidateVgpuBatchGPU(ids []string, deviceName string) ([]bool, error) {
	keep := make([]bool, len(ids))
	var raw [][]byte
	var at []int
	for i, id := range ids {
		data, err := os.ReadFile(filepath.Join(vGpuBasePath, id, "mdev_type/name"))
		if err != nil {
			continue
		}
		raw = append(raw, data)
		at = append(at, i)
	}
	if len(raw) == 0 {
		return keep, nil
	}
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return nil, err
	}
	dict, freeDict := cTypeDict(raw)
	defer freeDict()
	match := (*C.uint8_t)(C.malloc(C.size_t(len(raw))))
	defer C.free(unsafe.Pointer(match))
	var name *C.uint8_t
	if len(deviceName) > 0 {
		cname := C.CString(deviceName)
		defer C.free(unsafe.Pointer(cname))
		name = (*C.uint8_t)(unsafe.Pointer(cname))
	}
	if rc := C.kvg_mdev_label_match(kvgCtx, &dict, name, C.size_t(len(deviceName)), match); rc != C.KVG_OK {
		return nil, fmt.Errorf("kvg_mdev_label_match: %s", C.GoString(C.kvg_last_error(kvgCtx)))
	}
	for k, m := range unsafe.Slice(match, len(raw)) {
		keep[at[k]] = m != 0
	}
	return keep, nil
}

// EGMEntryRaw is one entry of the EGM class directory as discoverEGMDevicesFunc's reads returned it, undecoded.
type EGMEntryRaw struct {
	Name       string
	GPUDevices []byte
	GPUErr     error // the gpu_devices read
	StatErr    error // os.Stat of /dev/<name>
}

// discoverEGMRaw lists and reads what discoverEGMDevicesFunc (generic_device_plugin.go:120-157) reads, for every
// entry, and decodes nothing: kvg_pci_allocate_raw applies the "egm" prefix, strings.Fields and the Stat rule.
func discoverEGMRaw() ([]EGMEntryRaw, error) {
	egmClassDir := filepath.Join(rootPath, strings.TrimPrefix(egmClassPath, "/"))
	entries, err := os.ReadDir(egmClassDir)
	if err != nil {
		if errors.Is(err, fs.ErrNotExist) {
			return nil, nil
		}
		return nil, err
	}
	out := make([]EGMEntryRaw, 0, len(entries))
	for _, entry := range entries {
		e := EGMEntryRaw{Name: entry.Name()}
		e.GPUDevices, e.GPUErr = os.ReadFile(filepath.Join(egmClassDir, e.Name, "gpu_devices"))
		_, e.StatErr = os.Stat(filepath.Join(rootPath, strings.TrimPrefix(filepath.Join(deviceDir, e.Name), "/")))
		out = append(out, e)
	}
	return out, nil
}

// allocateRawGPU is allocateCheckGPU with no decoding in Go (Python twin: kvgpu/serve.py AllocateRawCheck, tested
// against AllocateCheck by tests/test_serve_allocate_raw.py): every member's iommu_group link target and vendor
// contents are read raw with os.Readlink and os.ReadFile, and together with the group string the maps hold, the
// DevicesIDs and discoverEGMRaw's entries go to one kvg_pci_allocate_raw call, which applies readLinkFunc,
// readIDFromFileFunc, discoverEGMDevicesFunc and egmPathsForAllocatedGPUs' key rule on the GPU.  Where the library
// reports that the reference's vendor read panics (panic[r]), vendorPanic re-slices the same bytes, so d.panic is the
// runtime.Error the reference's data[2:] raises, the value allocateCheckGPU recovers.  Like the rest of the file it
// is source only and has not been compiled.
func allocateRawGPU(members [][]allocMember, ids [][]string, egm []EGMEntryRaw) ([]allocDecision, error) {
	if len(members) == 0 && len(egm) == 0 {
		return nil, nil
	}
	var mOff, iOff, eOff []uint32
	var mBytes, iBytes, eBytes []byte
	var mState, eState []uint16
	var vendors [][]byte // per member, the vendor contents as read
	push := func(off *[]uint32, b *[]byte, data []byte) {
		if len(*off) == 0 {
			*off = append(*off, 0)
		}
		*b = append(*b, data...)
		*off = append(*off, uint32(len(*b)))
	}
	reqs := make([]C.kvg_alloc_req, len(members))
	for r := range members {
		for _, m := range members[r] {
			st := uint16(1<<C.KVG_AMEM_LINK | 1<<C.KVG_AMEM_VENDOR)
			target, err := os.Readlink(filepath.Join(basePath, m.addr, "iommu_group"))
			if err != nil {
				st |= 1 << (8 + C.KVG_AMEM_LINK)
			}
			vendor, err := os.ReadFile(filepath.Join(basePath, m.addr, "vendor"))
			if err != nil {
				st |= 1 << (8 + C.KVG_AMEM_VENDOR)
			}
			push(&mOff, &mBytes, []byte(target))
			push(&mOff, &mBytes, vendor)
			push(&mOff, &mBytes, []byte(m.group))
			mState = append(mState, st)
			vendors = append(vendors, vendor)
		}
		for _, id := range ids[r] {
			push(&iOff, &iBytes, []byte(id))
		}
		reqs[r] = C.kvg_alloc_req{n_members: C.uint32_t(len(members[r])), n_ids: C.uint32_t(len(ids[r]))}
	}
	for _, e := range egm {
		st := uint16(1<<C.KVG_AEGM_GPUS | 1<<C.KVG_AEGM_STAT)
		if e.GPUErr != nil {
			st |= 1 << (8 + C.KVG_AEGM_GPUS)
		}
		if e.StatErr != nil {
			st |= 1 << (8 + C.KVG_AEGM_STAT)
		}
		push(&eOff, &eBytes, []byte(e.Name))
		push(&eOff, &eBytes, e.GPUDevices)
		eState = append(eState, st)
	}
	// the library copies the inputs before it returns (cgo pointer rule): C copies of every table and byte array, so
	// &raw, a Go value, holds no Go pointer
	var cmem []unsafe.Pointer
	defer func() {
		for _, p := range cmem {
			C.free(p)
		}
	}()
	cCopy := func(b []byte) unsafe.Pointer {
		if len(b) == 0 {
			return nil
		}
		p := C.CBytes(b)
		cmem = append(cmem, p)
		return p
	}
	u32 := func(v []uint32) *C.uint32_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint32_t)(cCopy(unsafe.Slice((*byte)(unsafe.Pointer(&v[0])), 4*len(v))))
	}
	u16 := func(v []uint16) *C.uint16_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint16_t)(cCopy(unsafe.Slice((*byte)(unsafe.Pointer(&v[0])), 2*len(v))))
	}
	var raw C.kvg_alloc_raw
	raw.n_members = C.size_t(len(mState))
	raw.member_off, raw.member_state = u32(mOff), u16(mState)
	raw.member_bytes = (*C.uint8_t)(cCopy(mBytes))
	if len(iOff) > 0 {
		raw.n_ids = C.size_t(len(iOff) - 1)
	}
	raw.id_off, raw.id_bytes = u32(iOff), (*C.uint8_t)(cCopy(iBytes))
	raw.n_egm = C.uint32_t(len(egm))
	raw.egm_off, raw.egm_state = u32(eOff), u16(eState)
	raw.egm_bytes = (*C.uint8_t)(cCopy(eBytes))
	firstBad := make([]C.uint32_t, len(members)+1)
	panics := make([]C.uint8_t, len(members)+1)
	kept := make([]C.uint8_t, len(egm)+1)
	take := make([]C.uint8_t, len(members)*len(egm)+1)
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return nil, err
	}
	var reqPtr *C.kvg_alloc_req
	if len(reqs) > 0 {
		reqPtr = &reqs[0]
	}
	if rc := C.kvg_pci_allocate_raw(kvgCtx, reqPtr, C.uint32_t(len(reqs)), &raw, &firstBad[0], &panics[0], &kept[0],
		&take[0]); rc != C.KVG_OK {
		return nil, fmt.Errorf("kvg_pci_allocate_raw: %d %s", int(rc), C.GoString(C.kvg_last_error(kvgCtx)))
	}
	out := make([]allocDecision, len(members))
	for r, m0 := 0, 0; r < len(members); m0, r = m0+len(members[r]), r+1 {
		d := allocDecision{bad: -1, egm: []string{}}
		if int(firstBad[r]) < len(members[r]) {
			d.bad = int(firstBad[r])
			if panics[r] != 0 {
				d.panic = vendorPanic(vendors[m0+d.bad])
			}
		}
		for e := range egm { // ReadDir order is name order, so the paths come out sorted
			if kept[e] != 0 && take[r*len(egm)+e] != 0 {
				d.egm = append(d.egm, filepath.Join(deviceDir, egm[e].Name))
			}
		}
		out[r] = d
	}
	return out, nil
}

// vendorPanic is what readIDFromFileFunc's strings.Trim(string(data[2:]), "\n") panics with on `data`: the recovered
// runtime.Error, or nil when it does not panic.
func vendorPanic(data []byte) (p interface{}) {
	defer func() { p = recover() }()
	_ = strings.Trim(string(data[2:]), "\n")
	return nil
}

// allocVisit is one DevicesID a container request visits: the ID, the group bdfToIommu holds for it and that
// group's iommuMap members in map order.
type allocVisit struct {
	bdf, group string
	addrs      []string
}

// allocPlan is one container request's plan from the map lookups: its DevicesIDs, the IDs visited in order, and
// whether the ID after them misses the maps (the reference's first "unknown device" before any read).
type allocPlan struct {
	ids       []string
	visits    []allocVisit
	lookupErr bool
}

// allocateResponseGPU is the passthrough plugin's whole Allocate (generic_device_plugin.go:352-444) after the map
// lookups, in one kvg_pci_allocate_response call (Python twin: kvgpu/serve.py AllocateResponder, tested against the
// replay with AllocateRawCheck by tests/test_serve_allocate_response.py).  Every planned member's iommu_group link
// target, vendor contents and, with iommufd, vfio-dev listing (os.ReadDir; each entry's DirEntry.IsDir(), which does
// not follow links) are read raw; the library decides the re-check, readVFIODev, requestedDeviceFound, the device
// specs with appendDeviceSpec's de-duplication, the env value and the EGM paths.  Go formats the first failing
// request's error, re-raises a reported vendor panic as the runtime.Error vendorPanic recovers from the same bytes,
// and otherwise builds the ContainerAllocateResponses.  iommufd is supportsIOMMUFD's result; its other errors stay
// with the caller.  Like the rest of the file it is source only and has not been compiled.
func allocateResponseGPU(deviceName string, plans []allocPlan, iommufd bool, egm []EGMEntryRaw) ([]*pluginapi.ContainerAllocateResponse, error) {
	if len(plans) == 0 && len(egm) == 0 {
		return nil, nil
	}
	var mOff, iOff, eOff, aOff, vFirst, vOff []uint32
	var mBytes, iBytes, eBytes, aBytes, vBytes, vDir, vState []byte
	var mState, eState []uint16
	var vendors [][]byte   // per member, the vendor contents as read
	var listErrs []error   // per member, the listing's error
	var addrs [][]string   // per request, its members' addresses in order
	push := func(off *[]uint32, b *[]byte, data []byte) {
		if len(*off) == 0 {
			*off = append(*off, 0)
		}
		*b = append(*b, data...)
		*off = append(*off, uint32(len(*b)))
	}
	reqs := make([]C.kvg_alloc_req, len(plans))
	nVisited := make([]uint32, len(plans))
	lookup := make([]byte, len(plans))
	var idMembers []uint32
	vFirst = append(vFirst, 0)
	for r, p := range plans {
		var ra []string
		for _, v := range p.visits {
			idMembers = append(idMembers, uint32(len(v.addrs)))
			for _, addr := range v.addrs {
				st := uint16(1<<C.KVG_AMEM_LINK | 1<<C.KVG_AMEM_VENDOR)
				target, err := os.Readlink(filepath.Join(basePath, addr, "iommu_group"))
				if err != nil {
					st |= 1 << (8 + C.KVG_AMEM_LINK)
				}
				vendor, err := os.ReadFile(filepath.Join(basePath, addr, "vendor"))
				if err != nil {
					st |= 1 << (8 + C.KVG_AMEM_VENDOR)
				}
				push(&mOff, &mBytes, []byte(target))
				push(&mOff, &mBytes, vendor)
				push(&mOff, &mBytes, []byte(v.group))
				mState = append(mState, st)
				vendors = append(vendors, vendor)
				push(&aOff, &aBytes, []byte(addr))
				var lerr error
				ls := byte(0)
				if iommufd {
					ls = C.KVG_AVFIO_MADE
					entries, err := os.ReadDir(filepath.Join(basePath, addr, "vfio-dev"))
					if err != nil {
						ls |= C.KVG_AVFIO_FAILED
						lerr = err
					}
					for _, e := range entries {
						push(&vOff, &vBytes, []byte(e.Name()))
						d := byte(0)
						if e.IsDir() {
							d = 1
						}
						vDir = append(vDir, d)
					}
				}
				vState = append(vState, ls)
				vFirst = append(vFirst, uint32(len(vDir)))
				listErrs = append(listErrs, lerr)
				ra = append(ra, addr)
			}
		}
		for _, id := range p.ids {
			push(&iOff, &iBytes, []byte(id))
		}
		reqs[r] = C.kvg_alloc_req{n_members: C.uint32_t(len(ra)), n_ids: C.uint32_t(len(p.ids))}
		nVisited[r] = uint32(len(p.visits))
		if p.lookupErr {
			lookup[r] = 1
		}
		addrs = append(addrs, ra)
	}
	for _, e := range egm {
		st := uint16(1<<C.KVG_AEGM_GPUS | 1<<C.KVG_AEGM_STAT)
		if e.GPUErr != nil {
			st |= 1 << (8 + C.KVG_AEGM_GPUS)
		}
		if e.StatErr != nil {
			st |= 1 << (8 + C.KVG_AEGM_STAT)
		}
		push(&eOff, &eBytes, []byte(e.Name))
		push(&eOff, &eBytes, e.GPUDevices)
		eState = append(eState, st)
	}
	// C copies of every table and byte array (cgo pointer rule): &raw and &in, Go values, hold no Go pointer
	var cmem []unsafe.Pointer
	defer func() {
		for _, p := range cmem {
			C.free(p)
		}
	}()
	cCopy := func(b []byte) unsafe.Pointer {
		if len(b) == 0 {
			return nil
		}
		p := C.CBytes(b)
		cmem = append(cmem, p)
		return p
	}
	u32 := func(v []uint32) *C.uint32_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint32_t)(cCopy(unsafe.Slice((*byte)(unsafe.Pointer(&v[0])), 4*len(v))))
	}
	u16 := func(v []uint16) *C.uint16_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint16_t)(cCopy(unsafe.Slice((*byte)(unsafe.Pointer(&v[0])), 2*len(v))))
	}
	u8 := func(v []byte) *C.uint8_t { return (*C.uint8_t)(cCopy(v)) }
	var raw C.kvg_alloc_raw
	raw.n_members = C.size_t(len(mState))
	raw.member_off, raw.member_state, raw.member_bytes = u32(mOff), u16(mState), u8(mBytes)
	if len(iOff) > 0 {
		raw.n_ids = C.size_t(len(iOff) - 1)
	}
	raw.id_off, raw.id_bytes = u32(iOff), u8(iBytes)
	raw.n_egm = C.uint32_t(len(egm))
	raw.egm_off, raw.egm_state, raw.egm_bytes = u32(eOff), u16(eState), u8(eBytes)
	if len(vOff) == 0 {
		vOff = append(vOff, 0)
	}
	var in C.kvg_alloc_resp_in
	if iommufd {
		in.iommufd = 1
	}
	in.n_visited, in.lookup_error, in.id_members = u32(nVisited), u8(lookup), u32(idMembers)
	in.addr_off, in.addr_bytes = u32(aOff), u8(aBytes)
	in.vfio_first, in.vfio_off, in.vfio_bytes = u32(vFirst), u32(vOff), u8(vBytes)
	in.vfio_dir, in.vfio_state = u8(vDir), u8(vState)
	kvgMu.Lock()
	defer kvgMu.Unlock()
	if err := kvgEnsure(); err != nil {
		return nil, err
	}
	var reqPtr *C.kvg_alloc_req
	if len(reqs) > 0 {
		reqPtr = &reqs[0]
	}
	var res *C.kvg_alloc_resp
	if rc := C.kvg_pci_allocate_response(kvgCtx, reqPtr, C.uint32_t(len(reqs)), &raw, &in, &res); rc != C.KVG_OK {
		return nil, fmt.Errorf("kvg_pci_allocate_response: %d %s", int(rc), C.GoString(C.kvg_last_error(kvgCtx)))
	}
	defer C.kvg_result_free(unsafe.Pointer(res))
	n := len(plans)
	errKind := unsafe.Slice((*uint8)(unsafe.Pointer(res.error)), n)
	errAt := unsafe.Slice((*uint32)(unsafe.Pointer(res.error_at)), n)
	specFirst := unsafe.Slice((*uint32)(unsafe.Pointer(res.spec_first)), n)
	nSpecs := unsafe.Slice((*uint32)(unsafe.Pointer(res.n_specs)), n)
	envLen := unsafe.Slice((*uint32)(unsafe.Pointer(res.env_len)), n)
	envKey := unsafe.Slice((*uint8)(unsafe.Pointer(res.env_key)), n)
	key := fmt.Sprintf("%s_%s", gpuPrefix, strings.ToUpper(deviceName))
	out := make([]*pluginapi.ContainerAllocateResponse, 0, n)
	for r, m0 := 0, 0; r < n; m0, r = m0+len(addrs[r]), r+1 {
		at := int(errAt[r])
		switch errKind[r] {
		case C.KVG_ARESP_UNKNOWN_ID:
			return nil, fmt.Errorf("invalid allocation request: unknown device: %s", plans[r].ids[at])
		case C.KVG_ARESP_UNKNOWN_MEMBER:
			return nil, fmt.Errorf("invalid allocation request: unknown device: %s", addrs[r][at])
		case C.KVG_ARESP_PANIC:
			panic(vendorPanic(vendors[m0+at]))
		case C.KVG_ARESP_VFIO_READ:
			return nil, fmt.Errorf("could not determine iommufd device for device %s: %v", addrs[r][at], listErrs[m0+at])
		case C.KVG_ARESP_VFIO_NONE:
			return nil, fmt.Errorf("could not determine iommufd device for device %s: %v", addrs[r][at],
				errors.New("no iommufd device found"))
		}
		specs := make([]*pluginapi.DeviceSpec, 0, int(nSpecs[r]))
		spans := unsafe.Slice((*uint32)(unsafe.Pointer(res.spec_span)), 2*(int(specFirst[r])+int(nSpecs[r])))
		for s := int(specFirst[r]); s < int(specFirst[r])+int(nSpecs[r]); s++ {
			p := C.GoStringN((*C.char)(unsafe.Add(unsafe.Pointer(res.spec_bytes), spans[2*s])), C.int(spans[2*s+1]))
			specs = append(specs, &pluginapi.DeviceSpec{HostPath: p, ContainerPath: p, Permissions: "mrw"})
		}
		envs := map[string]string{}
		if envKey[r] != 0 {
			envs[key] = C.GoStringN((*C.char)(unsafe.Pointer(res.env_bytes)), C.int(envLen[r]))
		}
		out = append(out, &pluginapi.ContainerAllocateResponse{Envs: envs, Devices: specs})
	}
	return out, nil
}
