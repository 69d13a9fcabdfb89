"""ctypes binding of libkvgpu.so — exactly the symbols include/kvgpu.h declares.

There is no CPU fallback: if the library is missing or no CUDA device is usable, every compute
entry point raises KvgError.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG, "libkvgpu.so")
HEADER_PATH = os.path.join(os.path.dirname(_PKG), "include", "kvgpu.h")

KVG_OK, KVG_EINVAL, KVG_ECUDA, KVG_ENOMEM, KVG_ENCCL, KVG_ESTATE, KVG_ERANGE = 0, -1, -2, -3, -4, -5, -6
KVG_EPANIC = -7
RAW_NAME, RAW_VENDOR, RAW_DRIVER, RAW_GROUP, RAW_NUMA, RAW_DEVICE, RAW_FIELDS = range(7)
MRAW_NAME, MRAW_TYPE, MRAW_LINK, MRAW_NUMA, MRAW_FIELDS = range(5)
AMEM_LINK, AMEM_VENDOR, AMEM_GROUP, AMEM_FIELDS = range(4)
AEGM_NAME, AEGM_GPUS, AEGM_FIELDS = range(3)
AEGM_STAT = AEGM_FIELDS
ARESP_OK, ARESP_UNKNOWN_ID, ARESP_UNKNOWN_MEMBER, ARESP_PANIC, ARESP_VFIO_READ, ARESP_VFIO_NONE = range(6)
AVFIO_MADE, AVFIO_FAILED = 1, 2
KVG_NO_NAME = 0xFFFFFFFF
ERR_NAMES = {0: "KVG_OK", -1: "KVG_EINVAL", -2: "KVG_ECUDA", -3: "KVG_ENOMEM", -4: "KVG_ENCCL",
             -5: "KVG_ESTATE", -6: "KVG_ERANGE", -7: "KVG_EPANIC"}

DRV_NONE, DRV_VFIO_PCI, DRV_NVGRACE, DRV_OTHER = 0, 1, 2, 3
PF_VENDOR_ERR, PF_DRIVER_ERR, PF_IOMMU_ERR, PF_DEVICE_ERR, PF_NUMA_ERR = 1, 2, 4, 8, 16
MF_TYPE_ERR, MF_PARENT_ERR, MF_NUMA_ERR = 1, 2, 4

PCI_REC = np.dtype([("addr", "<u4"), ("vendor", "<u2"), ("device", "<u2"), ("iommu_group", "<u4"),
                    ("driver", "u1"), ("flags", "u1"), ("numa", "<i2")])
PCI_SURV = np.dtype([("addr", "<u4"), ("iommu_group", "<u4"), ("device", "<u2"), ("numa", "<u2"),
                     ("name_slot", "<u4")])
MDEV_REC = np.dtype([("uuid", "u1", (16,)), ("parent", "<u4"), ("type_idx", "<u2"), ("flags", "u1"),
                     ("pad0", "u1"), ("parent_numa", "<i2"), ("pad1", "u1", (6,))])
MDEV_SURV = np.dtype([("uuid", "u1", (16,)), ("parent", "<u4"), ("type_key", "<u2"),
                      ("numa", "<u2"), ("src", "<u4"), ("pad", "<u4")])
PCI_CHANGE = np.dtype([("addr", "<u4"), ("what", "<u4"), ("prev_group", "<u4"), ("now_group", "<u4"),
                       ("prev_device", "<u2"), ("now_device", "<u2"), ("prev_numa", "<u2"), ("now_numa", "<u2"),
                       ("now_index", "<u4"), ("prev_index", "<u4")])
MDEV_CHANGE = np.dtype([("uuid", "u1", (16,)), ("what", "<u4"), ("prev_parent", "<u4"), ("now_parent", "<u4"),
                        ("prev_type", "<u2"), ("now_type", "<u2"), ("prev_numa", "<u2"), ("now_numa", "<u2"),
                        ("now_index", "<u4"), ("prev_index", "<u4"), ("pad", "<u4")])
CH_ADDED, CH_REMOVED, CH_GROUP, CH_DEVICE, CH_NUMA = 1, 2, 4, 8, 16
CH_TYPE, CH_PARENT = 32, 64
NO_INDEX = 0xFFFFFFFF
PREF_ID = np.dtype([("handle", "<u4"), ("node", "<u4")])
PREF_REQ = np.dtype([("n_must", "<u4"), ("n_avail", "<u4"), ("size", "<i4"), ("pad", "<u4")])
PREF_RES = np.dtype([("n_out", "<i4"), ("n_must_distinct", "<u4")])
PREF_NODE_NONE = 0xFFFFFFFF
ALLOC_REQ = np.dtype([("n_members", "<u4"), ("n_ids", "<u4")])
ALLOC_MAX_EGM_GPUS = 65536
ALLOC_RAW_MAX_EGM_KEYS = ALLOC_MAX_EGM_GPUS - 1
assert PCI_REC.itemsize == 16 and PCI_SURV.itemsize == 16 and PCI_CHANGE.itemsize == 32
assert MDEV_REC.itemsize == 32 and MDEV_SURV.itemsize == 32 and MDEV_CHANGE.itemsize == 48
assert PREF_ID.itemsize == 8 and PREF_REQ.itemsize == 16 and PREF_RES.itemsize == 8 and ALLOC_REQ.itemsize == 8


class KvgError(RuntimeError):
    def __init__(self, rc, msg):
        super().__init__("%s: %s" % (ERR_NAMES.get(rc, rc), msg))
        self.rc = rc


class TypeDict(C.Structure):
    _fields_ = [("n_types", C.c_uint32), ("off", C.POINTER(C.c_uint32)),
                ("bytes", C.POINTER(C.c_uint8))]


class PciResultC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_survivors", C.c_uint64),
                ("survivors", C.c_void_p),
                ("n_dev_keys", C.c_uint32), ("dev_keys", C.c_void_p), ("dev_off", C.c_void_p),
                ("dev_perm", C.c_void_p), ("dev_name_slot", C.c_void_p),
                ("n_groups", C.c_uint32), ("grp_keys", C.c_void_p), ("grp_off", C.c_void_p),
                ("grp_perm", C.c_void_p),
                ("name_pool", C.c_void_p), ("name_pool_len", C.c_size_t)]


class PciRawC(C.Structure):
    _fields_ = [("n", C.c_size_t), ("off", C.c_void_p), ("bytes", C.c_void_p), ("state", C.c_void_p)]


class AllocRawC(C.Structure):
    _fields_ = [("n_members", C.c_size_t), ("member_off", C.c_void_p), ("member_bytes", C.c_void_p),
                ("member_state", C.c_void_p), ("n_ids", C.c_size_t), ("id_off", C.c_void_p), ("id_bytes", C.c_void_p),
                ("n_egm", C.c_uint32), ("egm_off", C.c_void_p), ("egm_bytes", C.c_void_p), ("egm_state", C.c_void_p)]


class AllocRespInC(C.Structure):
    _fields_ = [("iommufd", C.c_uint32), ("n_visited", C.c_void_p), ("lookup_error", C.c_void_p),
                ("id_members", C.c_void_p), ("addr_off", C.c_void_p), ("addr_bytes", C.c_void_p),
                ("vfio_first", C.c_void_p), ("vfio_off", C.c_void_p), ("vfio_bytes", C.c_void_p),
                ("vfio_dir", C.c_void_p), ("vfio_state", C.c_void_p)]


class AllocRespC(C.Structure):
    _fields_ = [("n_reqs", C.c_uint32), ("error", C.c_void_p), ("error_at", C.c_void_p), ("spec_first", C.c_void_p),
                ("n_specs", C.c_void_p), ("spec_span", C.c_void_p), ("spec_bytes", C.c_void_p),
                ("env_len", C.c_void_p), ("env_key", C.c_void_p), ("env_bytes", C.c_void_p)]


class PciSnapC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("recs", C.c_void_p),
                ("packed_addr", C.c_uint8), ("groups_numeric", C.c_uint8), ("devices_numeric", C.c_uint8),
                ("n_group_names", C.c_uint32), ("group_off", C.c_void_p), ("group_bytes", C.c_void_p),
                ("n_device_names", C.c_uint32), ("device_off", C.c_void_p), ("device_bytes", C.c_void_p)]


class MdevRawC(C.Structure):
    _fields_ = [("n", C.c_size_t), ("off", C.c_void_p), ("bytes", C.c_void_p), ("state", C.c_void_p)]


class MdevSnapC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("recs", C.c_void_p), ("uuid_ok", C.c_uint8), ("parents_packed", C.c_uint8),
                ("n_types", C.c_uint32), ("type_off", C.c_void_p), ("type_bytes", C.c_void_p),
                ("n_parent_names", C.c_uint32), ("parent_off", C.c_void_p), ("parent_bytes", C.c_void_p)]


class MdevResultC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_survivors", C.c_uint64),
                ("survivors", C.c_void_p),
                ("n_type_keys", C.c_uint32), ("type_keys", C.c_void_p), ("type_off", C.c_void_p),
                ("type_perm", C.c_void_p),
                ("n_types", C.c_uint32), ("label_off", C.c_void_p), ("label_bytes", C.c_void_p),
                ("type_canon", C.c_void_p), ("type_name_off", C.c_void_p),
                ("type_name_bytes", C.c_void_p),
                ("n_parents", C.c_uint32), ("par_keys", C.c_void_p), ("par_off", C.c_void_p),
                ("par_perm", C.c_void_p)]


class PciShardResultC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_local", C.c_uint64), ("local", C.c_void_p),
                ("n_dev_members", C.c_uint64), ("dev_members", C.c_void_p),
                ("n_dev_keys", C.c_uint32), ("dev_keys", C.c_void_p), ("dev_off", C.c_void_p),
                ("dev_perm", C.c_void_p), ("dev_name_slot", C.c_void_p),
                ("n_grp_members", C.c_uint64), ("grp_members", C.c_void_p),
                ("n_groups", C.c_uint32), ("grp_keys", C.c_void_p), ("grp_off", C.c_void_p),
                ("grp_perm", C.c_void_p),
                ("name_pool", C.c_void_p), ("name_pool_len", C.c_size_t)]


class MdevShardResultC(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_local", C.c_uint64), ("local", C.c_void_p),
                ("n_type_members", C.c_uint64), ("type_members", C.c_void_p),
                ("n_type_keys", C.c_uint32), ("type_keys", C.c_void_p), ("type_off", C.c_void_p),
                ("type_perm", C.c_void_p),
                ("n_par_members", C.c_uint64), ("par_members", C.c_void_p),
                ("n_parents", C.c_uint32), ("par_keys", C.c_void_p), ("par_off", C.c_void_p),
                ("par_perm", C.c_void_p),
                ("n_types", C.c_uint32), ("label_off", C.c_void_p), ("label_bytes", C.c_void_p),
                ("type_canon", C.c_void_p), ("type_name_off", C.c_void_p),
                ("type_name_bytes", C.c_void_p)]


class HealthDeltaC(C.Structure):
    _fields_ = [("n_records", C.c_uint32), ("n_alive", C.c_uint32), ("n_changed", C.c_uint32),
                ("changed", C.c_void_p)]


class PciDeltaC(C.Structure):
    _fields_ = [("n_prev", C.c_uint64), ("n_changes", C.c_uint64), ("changes", C.c_void_p),
                ("n_dev_dirty", C.c_uint32), ("dev_dirty", C.c_void_p),
                ("n_dev_gone", C.c_uint32), ("dev_gone", C.c_void_p),
                ("n_grp_dirty", C.c_uint32), ("grp_dirty", C.c_void_p),
                ("n_grp_gone", C.c_uint32), ("grp_gone", C.c_void_p)]


class MdevDeltaC(C.Structure):
    _fields_ = [("n_prev", C.c_uint64), ("n_changes", C.c_uint64), ("changes", C.c_void_p),
                ("n_type_dirty", C.c_uint32), ("type_dirty", C.c_void_p),
                ("n_type_gone", C.c_uint32), ("type_gone_off", C.c_void_p), ("type_gone_bytes", C.c_void_p),
                ("n_par_dirty", C.c_uint32), ("par_dirty", C.c_void_p),
                ("n_par_gone", C.c_uint32), ("par_gone", C.c_void_p)]


def declared_symbols() -> list[str]:
    """Every function name include/kvgpu.h declares (used by the export test)."""
    src = open(HEADER_PATH).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(kvg_[a-z0-9_]+)\s*\(", src)))


_lib = None


def load() -> C.CDLL:
    """dlopen libkvgpu.so (built in-tree by __graft_entry__.build / csrc/Makefile)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KvgError(KVG_ECUDA, "libkvgpu.so is not built (%s); run `python -c 'import "
                       "__graft_entry__ as g; g.build()'` — there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, sz, u32, u64 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64
    P = C.POINTER
    sig = {
        "kvg_abi_version": (C.c_int, []),
        "kvg_ctx_create": (C.c_int, [C.c_int, P(vp)]),
        "kvg_ctx_destroy": (None, [vp]),
        "kvg_last_error": (C.c_char_p, [vp]),
        "kvg_result_free": (None, [vp]),
        "kvg_launch_count": (u64, [vp]),
        "kvg_stream": (vp, [vp]),
        "kvg_pciids_load": (C.c_int, [vp, vp, sz]),
        "kvg_name_lookup": (C.c_int, [vp, C.c_char_p, sz, C.c_char_p, sz, P(sz)]),
        "kvg_name_table": (C.c_int, [vp, u32, u32, vp, vp, sz]),
        "kvg_pciids_info": (C.c_int, [vp, P(u32), P(u32), P(u32), P(u32)]),
        "kvg_scan_pci": (C.c_int, [vp, vp, sz, P(P(PciResultC))]),
        "kvg_scan_pci_raw": (C.c_int, [vp, P(PciRawC), P(P(PciResultC)), P(P(PciSnapC))]),
        "kvg_scan_mdev": (C.c_int, [vp, vp, sz, P(TypeDict), P(P(MdevResultC))]),
        "kvg_scan_mdev_raw": (C.c_int, [vp, P(MdevRawC), P(P(MdevResultC)), P(P(MdevSnapC))]),
        "kvg_mdev_label_match": (C.c_int, [vp, P(TypeDict), vp, sz, vp]),
        "kvg_pci_group_check": (C.c_int, [vp, vp, vp, sz, P(sz)]),
        "kvg_preferred_allocation": (C.c_int, [vp, vp, u32, vp, sz, vp, vp]),
        "kvg_pci_allocate_check": (C.c_int, [vp, vp, u32, vp, vp, sz, vp, sz, vp, vp, u32, u32, vp, vp]),
        "kvg_pci_allocate_raw": (C.c_int, [vp, vp, u32, P(AllocRawC), vp, vp, vp, vp]),
        "kvg_pci_allocate_response": (C.c_int, [vp, vp, u32, P(AllocRawC), P(AllocRespInC), P(P(AllocRespC))]),
        "kvg_health_rescan": (C.c_int, [vp, vp, sz, P(P(HealthDeltaC))]),
        "kvg_health_reset": (C.c_int, [vp]),
        "kvg_health_rescan_mdev": (C.c_int, [vp, vp, sz, u32, vp, sz, P(P(HealthDeltaC))]),
        "kvg_health_mdev_reset": (C.c_int, [vp]),
        "kvg_health_rescan_groups": (C.c_int, [vp, vp, sz, vp, sz, P(P(HealthDeltaC))]),
        "kvg_health_groups_reset": (C.c_int, [vp]),
        "kvg_health_rescan_mdev_keyed": (C.c_int, [vp, vp, sz, u32, vp, sz, P(P(HealthDeltaC))]),
        "kvg_health_rescan_groups_keyed": (C.c_int, [vp, vp, sz, vp, sz, P(P(HealthDeltaC))]),
        "kvg_health_rescan_groups_raw": (C.c_int, [vp, P(PciRawC), P(TypeDict), P(P(HealthDeltaC))]),
        "kvg_health_rescan_mdev_raw": (C.c_int, [vp, P(MdevRawC), P(TypeDict), P(P(HealthDeltaC))]),
        "kvg_scan_pci_delta": (C.c_int, [vp, vp, sz, P(P(PciResultC)), P(P(PciDeltaC))]),
        "kvg_scan_pci_delta_reset": (C.c_int, [vp]),
        "kvg_scan_pci_raw_delta": (C.c_int, [vp, P(PciRawC), P(P(PciResultC)), P(P(PciSnapC)), P(P(PciDeltaC))]),
        "kvg_scan_pci_raw_delta_reset": (C.c_int, [vp]),
        "kvg_scan_mdev_raw_delta": (C.c_int, [vp, P(MdevRawC), P(P(MdevResultC)), P(P(MdevSnapC)),
                                              P(P(MdevDeltaC))]),
        "kvg_scan_mdev_raw_delta_reset": (C.c_int, [vp]),
        "kvg_scan_mdev_delta": (C.c_int, [vp, vp, sz, P(TypeDict), P(P(MdevResultC)), P(P(MdevDeltaC))]),
        "kvg_scan_mdev_delta_reset": (C.c_int, [vp]),
        "kvg_text_pad": (sz, [sz]),
        "kvg_dev_pciids_parse": (C.c_int, [vp, vp, sz, sz, u32]),
        "kvg_dev_scan_pci": (C.c_int, [vp, vp, sz]),
        "kvg_dev_scan_pci_fetch": (C.c_int, [vp, P(P(PciResultC))]),
        "kvg_dev_scan_pci_count": (C.c_int, [vp, P(u64), P(u32), P(u32)]),
        "kvg_dev_gen_pci": (C.c_int, [vp, vp, u64, sz, vp, u32, u32]),
        "kvg_dev_gen_mdev": (C.c_int, [vp, vp, u64, sz]),
        "kvg_dev_scan_mdev": (C.c_int, [vp, vp, sz, P(TypeDict)]),
        "kvg_dev_scan_mdev_fetch": (C.c_int, [vp, P(P(MdevResultC))]),
        "kvg_dev_flush_l2": (C.c_int, [vp]),
        "kvg_kernel_times": (C.c_int, [vp, P(C.c_float), C.c_char_p, sz, C.c_int]),
        "kvg_set_kernel_timing": (C.c_int, [vp, C.c_int]),
        "kvg_comm_unique_id": (C.c_int, [vp]),
        "kvg_comm_init": (C.c_int, [vp, C.c_int, C.c_int, vp]),
        "kvg_comm_destroy": (C.c_int, [vp]),
        "kvg_comm_p2p_export": (C.c_int, [vp, C.c_int, C.c_int, sz, vp]),
        "kvg_comm_p2p_import": (C.c_int, [vp, vp]),
        "kvg_comm_p2p_enable": (C.c_int, [vp, C.c_int]),
        "kvg_debug_radix_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp]),
        "kvg_dev_scan_pci_sharded": (C.c_int, [vp, vp, sz]),
        "kvg_dev_scan_pci_shard_fetch": (C.c_int, [vp, P(P(PciShardResultC))]),
        "kvg_dev_scan_pci_shard_fetch_delta": (C.c_int, [vp, P(P(PciShardResultC)), P(P(PciDeltaC))]),
        "kvg_dev_scan_pci_shard_delta_reset": (C.c_int, [vp]),
        "kvg_dev_scan_mdev_sharded": (C.c_int, [vp, vp, sz, P(TypeDict)]),
        "kvg_dev_scan_mdev_shard_fetch": (C.c_int, [vp, P(P(MdevShardResultC))]),
        "kvg_dev_scan_mdev_shard_fetch_delta": (C.c_int, [vp, P(P(MdevShardResultC)), P(P(MdevDeltaC))]),
        "kvg_dev_scan_mdev_shard_delta_reset": (C.c_int, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _arr(ptr, n, dtype):
    """copy n items of dtype out of a library-owned buffer"""
    if not n:
        return np.zeros(0, dtype=dtype)
    nbytes = int(n) * np.dtype(dtype).itemsize
    return np.frombuffer(C.string_at(ptr, nbytes), dtype=dtype).copy()
