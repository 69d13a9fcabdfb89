/*
 * kvgpu.h — C-ABI of libkvgpu.so: the H100 (sm_90a) discovery-and-classification scan
 * that replaces the CPU scan of NVIDIA/kubevirt-gpu-device-plugin.
 *
 * The reference has NO FFI on this path today (it is pure Go).  The seam a maintainer binds is
 * the reference's own injection points; each entry point below cites the reference function it
 * replaces (paths relative to the reference repo root):
 *
 *   kvg_pciids_load   + kvg_name_lookup   <- getDeviceName / locateVendor
 *                                            pkg/device_plugin/device_plugin.go:371-438
 *   kvg_scan_pci                          <- createIommuDeviceMap   device_plugin.go:187-247
 *                                            (+ isSupportedVfioDriver :249-252, name join :124-128)
 *   kvg_scan_mdev                         <- createVgpuIDMap        device_plugin.go:255-291
 *                                            (+ readVgpuIDFromFileFunc label rule :334-344, join :152-155)
 *   kvg_health_rescan                     <- health flips fed to ListAndWatch
 *                                            generic_device_plugin.go:325-342, :611-690
 *   kvg_scan_pci_delta                    <- (no reference equivalent: the reference never re-scans)
 *   kvg_scan_mdev_delta                   <- (no reference equivalent: createVgpuIDMap runs once)
 *   kvg_comm_*, kvg_scan_pci_sharded      <- (no reference equivalent; BASELINE.json config 4)
 *   kvg_dev_scan_pci_shard_fetch_delta    <- (no reference equivalent: the re-scan delta of the sharded scan)
 *   kvg_dev_scan_mdev_shard_fetch_delta   <- (no reference equivalent: the re-scan delta of the sharded vGPU scan)
 *
 * Plain C: pointers + sizes only, no C++ types, no exceptions cross this boundary.
 * Return value: 0 = KVG_OK, negative = error; text via kvg_last_error().
 * There is NO CPU fallback: without a usable CUDA device every compute call returns KVG_ECUDA.
 *
 * Threading: a kvg_ctx owns one CUDA stream and is single-threaded (caller serialises);
 * distinct contexts are independent.  The library never calls back into the caller and never
 * retains caller pointers after a call returns (cgo pointer rule): host inputs are copied into
 * pinned staging memory inside the call.  Result objects are library-owned, flat, pointer+length
 * arrays in host memory, valid until kvg_result_free().
 */
#ifndef KVGPU_H
#define KVGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KVG_ABI_VERSION 1

/* ---- error codes --------------------------------------------------------------------------- */
enum {
  KVG_OK = 0,
  KVG_EINVAL = -1, /* bad argument */
  KVG_ECUDA = -2,  /* CUDA runtime / no device / kernel failure */
  KVG_ENOMEM = -3, /* host or device allocation failed */
  KVG_ENCCL = -4,  /* NCCL not loadable or a collective failed */
  KVG_ESTATE = -5, /* call order (e.g. scan before kvg_pciids_load) */
  KVG_ERANGE = -6  /* output buffer too small / value does not fit the wire format */
};

/* ---- wire format ---------------------------------------------------------------------------- */

/* driver dictionary codes produced by the snapshotter (device_plugin.go:75-78, :212-220) */
enum {
  KVG_DRV_NONE = 0,   /* no driver link (readLink error; also sets KVG_PF_DRIVER_ERR) */
  KVG_DRV_VFIO_PCI = 1, /* "vfio-pci" */
  KVG_DRV_NVGRACE = 2,  /* "nvgrace_gpu_vfio_pci" */
  KVG_DRV_OTHER = 3     /* anything else; codes >= 3 are all "unsupported" */
};

/* kvg_pci_rec.flags: which sysfs read FAILED for this entry (device_plugin.go:202-238) */
enum {
  KVG_PF_VENDOR_ERR = 1u << 0, /* readIDFromFile(vendor) error   -> drop (:203-206) */
  KVG_PF_DRIVER_ERR = 1u << 1, /* readLink(driver) error         -> drop (:213-216) */
  KVG_PF_IOMMU_ERR = 1u << 2,  /* readLink(iommu_group) error    -> drop (:222-225) */
  KVG_PF_DEVICE_ERR = 1u << 3, /* readIDFromFile(device) error   -> drop (:235-238) */
  KVG_PF_NUMA_ERR = 1u << 4    /* readNUMANode error             -> numa 0, KEPT (:227-230) */
};

/* One PCI function as snapshotted from /sys/bus/pci/devices/<addr>/, 16 bytes = one uint4.
 * Records are stored in filepath.Walk order (ascending byte-wise entry name). */
typedef struct kvg_pci_rec {
  uint32_t addr;        /* address handle: packed BDF domain<<16|bus<<8|dev<<3|fn, or the Walk
                           index when the snapshot is in index mode (names kept by the host) */
  uint16_t vendor;      /* sysfs "vendor" as a number (0x10de = NVIDIA); strings that are not
                           "0x%04x" can never equal "10de" and are stored as 0xffff            */
  uint16_t device;      /* sysfs "device" as a number -> key "%04x"                            */
  uint32_t iommu_group; /* basename of the iommu_group link as a number (or interned id)       */
  uint8_t driver;       /* KVG_DRV_*                                                            */
  uint8_t flags;        /* KVG_PF_*                                                             */
  int16_t numa;         /* raw numa_node value (may be -1); ignored when KVG_PF_NUMA_ERR        */
} kvg_pci_rec;

/* One surviving (advertised) PCI function, 16 bytes.  Order = Walk order (stable compaction). */
typedef struct kvg_pci_surv {
  uint32_t addr;
  uint32_t iommu_group;
  uint16_t device;
  uint16_t numa;      /* clamped: negative or unreadable -> 0 (device_plugin.go:316-318, :227-230) */
  uint32_t name_slot; /* offset into the context's name pool, or KVG_NO_NAME (getDeviceName == "") */
} kvg_pci_surv;

#define KVG_NO_NAME 0xffffffffu

/* kvg_mdev_rec.flags (device_plugin.go:269-284) */
enum {
  KVG_MF_TYPE_ERR = 1u << 0,   /* readVgpuIDFromFile error -> drop (:270-273) */
  KVG_MF_PARENT_ERR = 1u << 1, /* readGpuIDForVgpu error   -> drop (:276-279) */
  KVG_MF_NUMA_ERR = 1u << 2    /* parent numa unreadable   -> 0, KEPT (:281-284) */
};

/* One mediated device from /sys/bus/mdev/devices/<uuid>, 32 bytes, Walk order. */
typedef struct kvg_mdev_rec {
  uint8_t uuid[16];    /* big-endian UUID bytes (index mode: bytes 0..3 = BE Walk index) */
  uint32_t parent;     /* parent GPU address handle (packed BDF or interned id)          */
  uint16_t type_idx;   /* index into the raw type-name dictionary                        */
  uint8_t flags;       /* KVG_MF_*                                                        */
  uint8_t pad0;
  int16_t parent_numa; /* raw numa_node of the parent (may be -1)                        */
  uint8_t pad1[6];
} kvg_mdev_rec;

/* One surviving mdev, 32 bytes, Walk order. */
typedef struct kvg_mdev_surv {
  uint8_t uuid[16];
  uint32_t parent;
  uint16_t type_key; /* canonical type id = smallest raw index with the same sanitised label */
  uint16_t numa;
  uint32_t src;      /* index of the source record */
  uint32_t pad;
} kvg_mdev_surv;

/* Raw mdev_type/name file contents, unsanitised (the GPU applies device_plugin.go:341-342). */
typedef struct kvg_type_dict {
  uint32_t n_types;
  const uint32_t *off; /* n_types+1 offsets into bytes */
  const uint8_t *bytes;
} kvg_type_dict;

/* ---- results (library-owned host memory; free with kvg_result_free) ----------------------- */

typedef struct kvg_pci_result {
  uint64_t n_records;
  uint64_t n_survivors;
  const kvg_pci_surv *survivors; /* [n_survivors] Walk order == bdfToIommuMap insertion order */
  /* deviceMap (device_plugin.go:240): keys ascending; members of key k are
     survivors[dev_perm[dev_off[k] .. dev_off[k+1])], in Walk order */
  uint32_t n_dev_keys;
  const uint16_t *dev_keys;
  const uint32_t *dev_off;  /* [n_dev_keys+1] */
  const uint32_t *dev_perm; /* [n_survivors] */
  const uint32_t *dev_name_slot; /* [n_dev_keys] name pool offset or KVG_NO_NAME */
  /* iommuMap (device_plugin.go:241-242): same encoding, keys ascending numerically */
  uint32_t n_groups;
  const uint32_t *grp_keys;
  const uint32_t *grp_off;  /* [n_groups+1] */
  const uint32_t *grp_perm; /* [n_survivors] */
  /* sanitised names produced by the GPU; entry at slot s: uint16 length, then the bytes */
  const uint8_t *name_pool;
  size_t name_pool_len;
} kvg_pci_result;

typedef struct kvg_mdev_result {
  uint64_t n_records;
  uint64_t n_survivors;
  const kvg_mdev_surv *survivors;
  /* vGpuMap (device_plugin.go:288): keyed by canonical type id */
  uint32_t n_type_keys;
  const uint16_t *type_keys;
  const uint32_t *type_off;
  const uint32_t *type_perm;
  /* sanitised label of every raw dictionary entry (GPU output), and the resource-name join
     (getDeviceName(label), device_plugin.go:152): slot or KVG_NO_NAME */
  uint32_t n_types;
  const uint32_t *label_off; /* [n_types+1] into label_bytes */
  const uint8_t *label_bytes;
  const uint16_t *type_canon; /* [n_types] canonical id of each raw entry */
  const uint32_t *type_name_off; /* [n_types+1] into type_name_bytes: sanitised pci.ids name or empty */
  const uint8_t *type_name_bytes;
  /* gpuVgpuMap (device_plugin.go:287): keyed by parent handle ascending */
  uint32_t n_parents;
  const uint32_t *par_keys;
  const uint32_t *par_off;
  const uint32_t *par_perm;
} kvg_mdev_result;

/* ---- results of the SHARDED scans (one process per GPU; BASELINE.json config 4) ---------------------
 * Rank r scans records [r*N/P, (r+1)*N/P).  Its survivors stay local (concatenating the ranks' `local`
 * lists in rank order is the global Walk-order list, i.e. bdfToIommuMap / the mdev list).  The two group-by
 * maps are partitioned BY KEY: rank r holds exactly the keys with key % nranks == r, with ALL their members
 * (from every shard, Walk order).  Key sets of different ranks are disjoint; their union is the global map. */
typedef struct kvg_pci_shard_result {
  uint64_t n_records;             /* records of this rank's shard */
  uint64_t n_local;
  const kvg_pci_surv *local;      /* [n_local] this shard's survivors, Walk order */
  /* deviceMap part: members of the device ids this rank owns; key k = dev_members[dev_perm[dev_off[k]..)] */
  uint64_t n_dev_members;
  const kvg_pci_surv *dev_members;
  uint32_t n_dev_keys;
  const uint16_t *dev_keys;
  const uint32_t *dev_off;
  const uint32_t *dev_perm;
  const uint32_t *dev_name_slot;
  /* iommuMap part */
  uint64_t n_grp_members;
  const kvg_pci_surv *grp_members;
  uint32_t n_groups;
  const uint32_t *grp_keys;
  const uint32_t *grp_off;
  const uint32_t *grp_perm;
  const uint8_t *name_pool;
  size_t name_pool_len;
} kvg_pci_shard_result;

typedef struct kvg_mdev_shard_result {
  uint64_t n_records;
  uint64_t n_local;
  const kvg_mdev_surv *local;     /* [n_local] this shard's surviving mdevs, Walk order */
  /* vGpuMap part: canonical type ids owned by this rank */
  uint64_t n_type_members;
  const kvg_mdev_surv *type_members;
  uint32_t n_type_keys;
  const uint16_t *type_keys;
  const uint32_t *type_off;
  const uint32_t *type_perm;
  /* gpuVgpuMap part: parent handles owned by this rank */
  uint64_t n_par_members;
  const kvg_mdev_surv *par_members;
  uint32_t n_parents;
  const uint32_t *par_keys;
  const uint32_t *par_off;
  const uint32_t *par_perm;
  /* the type dictionary as in kvg_mdev_result (every rank loads the same dictionary) */
  uint32_t n_types;
  const uint32_t *label_off;
  const uint8_t *label_bytes;
  const uint16_t *type_canon;
  const uint32_t *type_name_off;
  const uint8_t *type_name_bytes;
} kvg_mdev_shard_result;

/* Health transitions of one re-scan relative to the previous one (record order). */
typedef struct kvg_health_delta {
  uint32_t n_records;
  uint32_t n_alive;   /* records passing the classification predicate now */
  uint32_t n_changed;
  const uint32_t *changed; /* [n_changed] (record index << 1) | now_alive, ascending index */
} kvg_health_delta;

/* ---- re-scan delta (K7): what changed since the previous kvg_scan_pci_delta / kvg_scan_mdev_delta
 * (kvg_pci_delta also serves kvg_dev_scan_pci_shard_fetch_delta and kvg_mdev_delta
 * kvg_dev_scan_mdev_shard_fetch_delta, where "survivors" are the local shard's) */
enum {
  KVG_CH_ADDED = 1u << 0,   /* survives now, did not before                    */
  KVG_CH_REMOVED = 1u << 1, /* survived before, does not now                    */
  KVG_CH_GROUP = 1u << 2,   /* survives on both sides with another iommu group  (PCI)  */
  KVG_CH_DEVICE = 1u << 3,  /* ... another device id                            (PCI)  */
  KVG_CH_NUMA = 1u << 4,    /* ... another clamped NUMA node                    */
  KVG_CH_TYPE = 1u << 5,    /* ... another sanitised type label                 (mdev) */
  KVG_CH_PARENT = 1u << 6   /* ... another parent GPU handle                    (mdev) */
};

typedef struct kvg_pci_change { /* 32 bytes; one per address whose survivor differs */
  uint32_t addr;
  uint32_t what;                  /* KVG_CH_* */
  uint32_t prev_group, now_group; /* 0 on the absent side */
  uint16_t prev_device, now_device;
  uint16_t prev_numa, now_numa;   /* clamped, as in kvg_pci_surv */
  uint32_t now_index;  /* index into this result's survivors, or 0xffffffff (removed) */
  uint32_t prev_index; /* index into the previous delta scan's survivors, or 0xffffffff (added) */
} kvg_pci_change;

typedef struct kvg_pci_delta {
  uint64_t n_prev;    /* survivors of the previous result (0: first call / after reset) */
  uint64_t n_changes;
  const kvg_pci_change *changes; /* [n_changes] ascending addr */
  uint32_t n_dev_dirty;
  const uint32_t *dev_dirty; /* indices into res->dev_keys, ascending */
  uint32_t n_dev_gone;
  const uint16_t *dev_gone;  /* device ids of the previous result absent now, ascending */
  uint32_t n_grp_dirty;
  const uint32_t *grp_dirty; /* indices into res->grp_keys, ascending */
  uint32_t n_grp_gone;
  const uint32_t *grp_gone;  /* groups of the previous result absent now, ascending */
} kvg_pci_delta;

typedef struct kvg_mdev_change { /* 48 bytes; one per UUID whose survivor differs */
  uint8_t uuid[16];
  uint32_t what;                    /* KVG_CH_ADDED / REMOVED / NUMA / TYPE / PARENT */
  uint32_t prev_parent, now_parent; /* 0 on the absent side */
  uint16_t prev_type, now_type;     /* canonical ids in the previous / this result's dictionary */
  uint16_t prev_numa, now_numa;     /* clamped, as in kvg_mdev_surv */
  uint32_t now_index;  /* index into this result's survivors, or 0xffffffff (removed) */
  uint32_t prev_index; /* index into the previous delta scan's survivors, or 0xffffffff (added) */
  uint32_t pad;
} kvg_mdev_change;

typedef struct kvg_mdev_delta {
  uint64_t n_prev;    /* survivors of the previous result (0: first call / after reset) */
  uint64_t n_changes;
  const kvg_mdev_change *changes; /* [n_changes] ascending UUID (big-endian byte order) */
  uint32_t n_type_dirty;
  const uint32_t *type_dirty;     /* indices into res->type_keys, ascending */
  /* vGpuMap keys of the previous result absent now, as labels, in ascending previous canonical id:
     label g = type_gone_bytes[type_gone_off[g] .. type_gone_off[g+1]) */
  uint32_t n_type_gone;
  const uint32_t *type_gone_off;  /* [n_type_gone + 1] */
  const uint8_t *type_gone_bytes;
  uint32_t n_par_dirty;
  const uint32_t *par_dirty;      /* indices into res->par_keys, ascending */
  uint32_t n_par_gone;
  const uint32_t *par_gone;       /* parent handles of the previous result absent now, ascending */
} kvg_mdev_delta;

/* ---- context -------------------------------------------------------------------------------- */
typedef struct kvg_ctx kvg_ctx;

int kvg_abi_version(void);
int kvg_ctx_create(int cuda_device, kvg_ctx **out);
void kvg_ctx_destroy(kvg_ctx *ctx);
const char *kvg_last_error(kvg_ctx *ctx); /* ctx may be NULL: last create error */
void kvg_result_free(void *result);
/* kernels launched by this context since creation (bench.py "gpu_launches") */
uint64_t kvg_launch_count(kvg_ctx *ctx);
/* the context's cudaStream_t, for CUDA-event timing on the launching stream */
void *kvg_stream(kvg_ctx *ctx);

/* ---- pci.ids name table (getDeviceName, device_plugin.go:371-438) --------------------------- */

/* Parse `text` on the GPU: line split, vendor context, (vendor,device)->line hash, NVIDIA
 * section bounds, sanitised names.  Idempotent: a second call replaces the table.
 * Pageable `text` (Go, Python bytes): copied and published before the call returns.
 * Page-locked `text` (cudaHostAlloc / cudaHostRegister): the call only ENQUEUES copy + parse, so
 * that the next call's host-to-device traffic overlaps it; the buffer must stay valid, and a
 * table-capacity error is reported, by the first later call on `ctx` that consumes the table
 * (kvg_name_lookup / kvg_name_table / kvg_pciids_info / any scan). */
int kvg_pciids_load(kvg_ctx *ctx, const uint8_t *text, size_t len);

/* Exact getDeviceName(key) for ANY key bytes: "" (outlen 0) when not found.  4-lower-hex keys go
 * through the table; every other key through the prefix-match kernel (device_plugin.go:388-400). */
int kvg_name_lookup(kvg_ctx *ctx, const char *key, size_t keylen, char *out, size_t cap,
                    size_t *outlen);

/* Bulk form used by tests and the Go shim: names of device ids [first, first+count) through the
 * table path; out_off has count+1 entries into out_bytes (cap bytes). */
int kvg_name_table(kvg_ctx *ctx, uint32_t first, uint32_t count, uint32_t *out_off,
                   uint8_t *out_bytes, size_t cap);

/* table facts after load: byte offsets of the first "10de" line and of the section end,
 * number of (vendor,device) entries inserted, number of text lines */
int kvg_pciids_info(kvg_ctx *ctx, uint32_t *vendor_off, uint32_t *section_end, uint32_t *n_entries,
                    uint32_t *n_lines);

/* ---- scans, host buffers in / host results out (the reference-facing calls) ---------------- */
int kvg_scan_pci(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n, kvg_pci_result **res);
/* (128 Ki <= n <= 16 Mi records: the snapshot is copied, classified and its survivors returned
 *  chunk by chunk on separate copy streams; results are identical.  KVG_PIPELINE=0 disables.) */
int kvg_scan_mdev(kvg_ctx *ctx, const kvg_mdev_rec *recs, size_t n, const kvg_type_dict *types,
                  kvg_mdev_result **res);
/* Classify `recs`, diff against the alive-set of the previous call on this context (first call:
 * against "nothing alive").  A call with a different n re-arms the same way, as does
 * kvg_health_reset(); n = 0 returns an empty delta.  Pinned (cudaHostAlloc / registered) `recs` of
 * at most 32,768 records are read in place by TMA bulk copies and must be 16-byte aligned; this is
 * not checked.  Pageable memory is staged and has no alignment requirement. */
int kvg_health_rescan(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n, kvg_health_delta **delta);
int kvg_health_reset(kvg_ctx *ctx);

/* Scan `recs` and diff the result against the previous one, keyed by survivor address.
 *
 * *res is byte for byte what kvg_scan_pci(ctx, recs, n, ...) returns for the same input, at every size (single
 * copy, pipelined, split classify and final steps).  *res and *delta are both freed with kvg_result_free.
 *
 * "Previous" is the result of the last SUCCESSFUL kvg_scan_pci_delta on this context since kvg_ctx_create or
 * kvg_scan_pci_delta_reset; before any such call it is empty, so every survivor is KVG_CH_ADDED, every key is dirty
 * and nothing is gone.  The library keeps its own copy of it: kvg_scan_pci, kvg_dev_scan_pci*, the mdev scans,
 * kvg_health_rescan, the sharded scans and kvg_pciids_load in between leave it unchanged.
 *
 * changes: an address has an entry iff it survives on exactly one side, or on both with a different iommu group,
 * device id or clamped NUMA node.  The name slot is not compared (a pci.ids reload is the caller's own event).
 * dev_dirty / grp_dirty: key k of deviceMap (iommuMap) is dirty iff the sequence of (addr, numa) of its members, in
 * Walk order, differs between the two results; keys that are new are dirty.  So a group-only change dirties
 * iommuMap keys and no deviceMap key, a device-only change deviceMap keys and no group, a NUMA change the key of
 * the device and the key of the group.  dev_gone / grp_gone: keys present before and absent now.
 *
 * Precondition: survivor addresses ascend strictly, and a handle means the same device in both snapshots.
 * Numeric (packed-BDF) snapshots satisfy both.  Strict ascent is checked on the device: if it fails the call
 * returns KVG_EINVAL (text in kvg_last_error), hands out no objects, and the previous result stays as it was.
 * Index-mode handles ascend but are not stable across snapshots: such calls are accepted, and the delta is then
 * relative to the handles only (a device that moved in the Walk shows as changed or as removed + added).
 *
 * Cost beyond kvg_scan_pci on the same input: two kernel launches and one synchronisation. */
int kvg_scan_pci_delta(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n, kvg_pci_result **res,
                       kvg_pci_delta **delta);
/* forget the previous result: the next kvg_scan_pci_delta reports everything as added */
int kvg_scan_pci_delta_reset(kvg_ctx *ctx);

/* Scan mdev `recs` with dictionary `types` and diff the result against the previous one, keyed by survivor UUID.
 *
 * *res is byte for byte what kvg_scan_mdev(ctx, recs, n, types, ...) returns for the same input, dictionary arrays
 * included.  *res and *delta are both freed with kvg_result_free.
 *
 * "Previous" is the result of the last SUCCESSFUL kvg_scan_mdev_delta on this context since kvg_ctx_create or
 * kvg_scan_mdev_delta_reset; before any such call it is empty, so every survivor is KVG_CH_ADDED, every key is dirty
 * and nothing is gone.  The library keeps its own copy of it, survivors, keys and type labels, separate from the PCI
 * delta's: kvg_scan_mdev, kvg_scan_pci, kvg_scan_pci_delta (and its reset), the kvg_dev_scan_* calls, the health
 * calls, the sharded scans and kvg_pciids_load in between leave it unchanged, and this call leaves the PCI delta's
 * previous result unchanged.
 *
 * Type identity across the two scans is the sanitised label, not the canonical id: each result numbers its own
 * dictionary (first appearance in the Walk), so one new raw name can renumber every later one, and raw names that
 * sanitise to one label are one key.
 *
 * changes: a UUID has an entry iff it survives on exactly one side, or on both with a different label
 * (KVG_CH_TYPE), parent handle (KVG_CH_PARENT) or clamped NUMA node (KVG_CH_NUMA).  `src` and the resource-name join
 * are not compared.  type_dirty: vGpuMap key (label) k is dirty iff the sequence of (uuid, numa) of its members, in
 * Walk order, differs between the two results; keys that are new are dirty.  par_dirty: gpuVgpuMap key k is dirty
 * iff its uuid sequence differs (its members carry no NUMA node, device_plugin.go:287-288).  So a NUMA-only change
 * dirties a vGpuMap key and no gpuVgpuMap key, and a parent-only change gpuVgpuMap keys only.  type_gone (labels) /
 * par_gone: keys present before and absent now; a label still in the dictionary without a survivor is gone.
 *
 * Precondition: survivor UUIDs ascend strictly (big-endian byte order), and a parent handle means the same GPU in
 * both snapshots.  Canonical UUID names and packed-BDF parents satisfy both.  Strict ascent is checked on the device:
 * if it fails the call returns KVG_EINVAL (text in kvg_last_error), hands out no objects, and the previous result
 * stays as it was; so does every error of the scan itself, e.g. KVG_ERANGE for more than 65,535 types.  Index-mode
 * UUIDs (Walk indices) and interned parents are accepted, but the delta is then relative to the handles only.
 *
 * Cost beyond kvg_scan_mdev on the same input: three kernel launches and one synchronisation. */
int kvg_scan_mdev_delta(kvg_ctx *ctx, const kvg_mdev_rec *recs, size_t n, const kvg_type_dict *types,
                        kvg_mdev_result **res, kvg_mdev_delta **delta);
/* forget the previous result: the next kvg_scan_mdev_delta reports everything as added */
int kvg_scan_mdev_delta_reset(kvg_ctx *ctx);

/* ---- device-resident entry points (inputs already in HBM; used by bench.py "value") -------- */

/* Layout contract for device text: 16-byte aligned `d_text`, 16 readable bytes BEFORE it and
 * kvg_text_pad(len) readable bytes from it, all padding bytes '\n'.  n_files images of `len`
 * bytes each, image f at d_text + f*stride (stride % 16 == 0, stride >= kvg_text_pad(len)+16).
 * Image 0 becomes the context's table; images >= 1 are parsed into scratch tables (batch
 * throughput measurement: every byte is split, every line start classified).
 * The first call on an image publishes its table (synchronous).  A later call on the SAME single image
 * re-parses it asynchronously on the context's side stream: it starts when everything enqueued before it
 * has finished, kvg_dev_scan_pci / kvg_dev_scan_pci_sharded enqueued after it classify and sort beside
 * it and join the names in their last kernel, every other consumer of the table waits for it first.
 * d_text must stay valid until the next call on the context that synchronises (any fetch / count). */
size_t kvg_text_pad(size_t len);
int kvg_dev_pciids_parse(kvg_ctx *ctx, const void *d_text, size_t len, size_t stride,
                         uint32_t n_files);
/* enqueue classify + stable compaction + both bucketings on the context stream; no host sync */
int kvg_dev_scan_pci(kvg_ctx *ctx, const void *d_recs, size_t n);
/* synchronise, copy the result of the last kvg_dev_scan_pci to the host */
int kvg_dev_scan_pci_fetch(kvg_ctx *ctx, kvg_pci_result **res);
/* survivor count of the last enqueued scan (synchronises the stream) */
int kvg_dev_scan_pci_count(kvg_ctx *ctx, uint64_t *n_survivors, uint32_t *n_dev_keys,
                           uint32_t *n_groups);
/* synthetic snapshot generators (counter-based splitmix64; oracle/kvg_oracle.c has the CPU twin) */
int kvg_dev_gen_pci(kvg_ctx *ctx, void *d_recs, uint64_t first, size_t n, const uint16_t *nv_ids,
                    uint32_t n_nv_ids, uint32_t group_bits);
int kvg_dev_gen_mdev(kvg_ctx *ctx, void *d_recs, uint64_t first, size_t n);
int kvg_dev_scan_mdev(kvg_ctx *ctx, const void *d_recs, size_t n, const kvg_type_dict *types);
int kvg_dev_scan_mdev_fetch(kvg_ctx *ctx, kvg_mdev_result **res);
/* Diagnostics: the pass structure (count, shift and width of each pass) the radix kernels derive on
 * the device for an ordering whose largest key is `max_key` (key_bits_max 16 or 32; max_bits 11, or 8 for
 * inputs >= 8 Mi records): pass 0 always takes the low max_bits bits, the remaining key bits are split
 * evenly over the fewest further passes.  Pure host arithmetic: usable without a GPU. */
int kvg_debug_radix_plan(uint32_t max_key, uint32_t key_bits_max, uint32_t max_bits, uint32_t *npass,
                         uint32_t *shifts4, uint32_t *bits4);

/* write `bytes` of zeros through a scratch buffer larger than L2 (timing hygiene, untimed) */
int kvg_dev_flush_l2(kvg_ctx *ctx);
/* per-kernel device time of the last kvg_dev_scan_pci / kvg_dev_pciids_parse, CUDA events on the
 * context stream; names is a NUL-separated list; returns count */
int kvg_kernel_times(kvg_ctx *ctx, float *ms, char *names, size_t names_cap, int max_n);
int kvg_set_kernel_timing(kvg_ctx *ctx, int enabled);

/* ---- multi-GPU (BASELINE.json config 4): one process per GPU, records range-sharded --------- */
#define KVG_UNIQUE_ID_BYTES 128
int kvg_comm_unique_id(void *out128);
int kvg_comm_init(kvg_ctx *ctx, int rank, int nranks, const void *unique_id128);
int kvg_comm_destroy(kvg_ctx *ctx);
/* Peer-memory exchange (CUDA IPC over NVLink, one process per GPU of ONE node): export allocates this
 * rank's receive window for shards of up to cap_local PCI records (cap_local / 2 mdev records) and returns
 * a 64-byte handle; import opens all ranks' handles (nranks x 64 bytes, rank order).  Afterwards the sharded
 * scans exchange by storing into the owners' windows and need neither NCCL nor a host synchronisation.
 * If either call fails the NCCL path (kvg_comm_init) remains usable. */
int kvg_comm_p2p_export(kvg_ctx *ctx, int rank, int nranks, size_t cap_local, void *handle_out64);
int kvg_comm_p2p_import(kvg_ctx *ctx, const void *all_handles);
/* collective decision: enable only when import succeeded on every rank */
int kvg_comm_p2p_enable(kvg_ctx *ctx, int on);
/* Classify the local shard (device memory), send every survivor to the owner of its key (once per
 * group-by map: key % nranks), order the owned members.  Peer windows: the multisplit stores straight into
 * the owners' windows over NVLink, nothing returns to the host.  NCCL mode: one allgatherv of the survivor
 * lists (two host synchronisations for the counts), then the same kernels keep what this rank owns.
 * Collective: every rank of the communicator must call it, in the same order. */
int kvg_dev_scan_pci_sharded(kvg_ctx *ctx, const void *d_recs, size_t n_local);
int kvg_dev_scan_pci_shard_fetch(kvg_ctx *ctx, kvg_pci_shard_result **res);
/* Fetch the last kvg_dev_scan_pci_sharded like kvg_dev_scan_pci_shard_fetch, and diff it against the previous
 * successful call of this function on this context: this rank's share of the re-scan delta of the whole snapshot.
 *
 * *res is byte for byte what kvg_dev_scan_pci_shard_fetch returns for the same scan.  *res and *delta are both freed
 * with kvg_result_free.  The call is NOT collective: it reads nothing from peers.
 *
 * "Previous" is the result of the last SUCCESSFUL call of this function on this context since kvg_ctx_create or
 * kvg_dev_scan_pci_shard_delta_reset; before any such call it is empty, so every local survivor is KVG_CH_ADDED,
 * every owned key is dirty and nothing is gone.  The library keeps its own copy of it (the local survivors, both
 * owned member lists and both owned key lists), separate from the other deltas': kvg_dev_scan_pci_shard_fetch, the
 * other scans, the other deltas and their resets, the health calls, kvg_pciids_load and the mdev sharded scan in
 * between leave it unchanged, and this call leaves theirs unchanged.
 *
 * changes: the local shard's survivors (res->local), keyed by address and in ascending address order, diffed against
 * the previous local list by the rules of kvg_scan_pci_delta.  now_index / prev_index index res->local / the previous
 * local list, and n_prev is the previous local count.  An address that crossed a shard boundary between the two
 * scans shows as KVG_CH_REMOVED on one rank and KVG_CH_ADDED on another; merging the ranks' changes in address order
 * and fusing such pairs gives exactly the kvg_scan_pci_delta of the concatenated snapshot.
 *
 * dev_dirty / grp_dirty: indices into res->dev_keys / res->grp_keys, the keys this rank owns (key % nranks == rank),
 * by the rule of kvg_scan_pci_delta: the (addr, numa) sequence of the key's members, in Walk order, changed.  The
 * owner of a key does not change between scans and the owned member lists hold every member from every shard, so
 * diffing them gives exactly this rank's share of the global lists, with no communication; a member that moved to a
 * key another rank owns is removed here and added there.  dev_gone / grp_gone: owned keys present before and absent
 * now.
 *
 * Precondition: survivor addresses ascend strictly in global Walk order (shards in rank order), and a handle means
 * the same device in both snapshots.  The local list and both owned member lists are checked for strict ascent on the
 * device: if that fails the call returns KVG_EINVAL (text in kvg_last_error), hands out no objects, and the previous
 * result stays as it was; so does every error of the fetch itself (e.g. KVG_ENCCL when a peer timed out).
 * KVG_EINVAL when the last scan on the context was not kvg_dev_scan_pci_sharded.
 *
 * Cost beyond kvg_dev_scan_pci_shard_fetch: two kernel launches and one synchronisation. */
int kvg_dev_scan_pci_shard_fetch_delta(kvg_ctx *ctx, kvg_pci_shard_result **res, kvg_pci_delta **delta);
/* forget the previous result: the next kvg_dev_scan_pci_shard_fetch_delta reports everything as added */
int kvg_dev_scan_pci_shard_delta_reset(kvg_ctx *ctx);
/* the same for mdev records (createVgpuIDMap): type / parent orderings of the owned members */
int kvg_dev_scan_mdev_sharded(kvg_ctx *ctx, const void *d_recs, size_t n_local, const kvg_type_dict *types);
int kvg_dev_scan_mdev_shard_fetch(kvg_ctx *ctx, kvg_mdev_shard_result **res);
/* Fetch the last kvg_dev_scan_mdev_sharded like kvg_dev_scan_mdev_shard_fetch, and diff it against the previous
 * successful call of this function on this context: this rank's share of the re-scan delta of the whole snapshot.
 *
 * *res is byte for byte what kvg_dev_scan_mdev_shard_fetch returns for the same scan.  *res and *delta are both freed
 * with kvg_result_free.  The call is NOT collective: it reads nothing from peers.
 *
 * "Previous" is the result of the last SUCCESSFUL call of this function on this context since kvg_ctx_create or
 * kvg_dev_scan_mdev_shard_delta_reset; before any such call it is empty, so every local survivor is KVG_CH_ADDED,
 * every owned key is dirty and nothing is gone.  The library keeps its own copy of it (the local survivors, both
 * owned member lists, both owned key lists, the dictionary's labels and its canonical ids), separate from the other
 * deltas': kvg_dev_scan_mdev_shard_fetch, the other scans, kvg_scan_mdev_delta, kvg_scan_pci_delta,
 * kvg_dev_scan_pci_shard_fetch_delta and their resets, the health calls and kvg_pciids_load in between leave it
 * unchanged, and this call leaves theirs unchanged.
 *
 * changes: the local shard's survivors (res->local), keyed by UUID and in ascending UUID order, diffed against the
 * previous local list by the rules of kvg_scan_mdev_delta; type identity is the sanitised label.  A local survivor's
 * type may be a label another rank owns, so the labels of every canonical id of both dictionaries are translated, not
 * only this rank's keys.  now_index / prev_index index res->local / the previous local list, and n_prev is the
 * previous local count.  A UUID that crossed a shard boundary between the two scans shows as KVG_CH_REMOVED on one
 * rank and KVG_CH_ADDED on another; merging the ranks' changes in UUID order and fusing such pairs gives exactly the
 * changes of kvg_scan_mdev_delta on the concatenated snapshot.
 *
 * type_dirty / type_gone / par_dirty / par_gone: the key rules of kvg_scan_mdev_delta applied to this rank's previous
 * and new OWNED member lists.  type_dirty indexes res->type_keys, par_dirty res->par_keys; type_gone holds labels and
 * par_gone parent handles.  A parent handle's owner never changes, so the par lists are exactly this rank's share of
 * the global lists.  A vGpuMap key is owned by canonical id % nranks in each scan's own dictionary: when the
 * dictionary renumbers, a label can move to another rank.  It is then in type_gone on its old owner and dirty on its
 * new one, even if its members did not change, which is what a server per rank must do (stop serving the label
 * here, start serving it there).  Outside such moves the type lists are exactly this rank's share of the global lists;
 * the global ones follow from the merged changes alone (a key is dirty iff some merged change touches it).
 *
 * Precondition: survivor UUIDs ascend strictly in global Walk order (shards in rank order), and a parent handle means
 * the same GPU in both snapshots.  The local list and both owned member lists are checked for strict ascent on the
 * device: if that fails the call returns KVG_EINVAL (text in kvg_last_error), hands out no objects, and the previous
 * result stays as it was; so does every error of the fetch itself (e.g. KVG_ENCCL when a peer timed out).  KVG_EINVAL
 * when the last scan on the context was not kvg_dev_scan_mdev_sharded.
 *
 * Cost beyond kvg_dev_scan_mdev_shard_fetch: three kernel launches and one synchronisation. */
int kvg_dev_scan_mdev_shard_fetch_delta(kvg_ctx *ctx, kvg_mdev_shard_result **res, kvg_mdev_delta **delta);
/* forget the previous result: the next kvg_dev_scan_mdev_shard_fetch_delta reports everything as added */
int kvg_dev_scan_mdev_shard_delta_reset(kvg_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* KVGPU_H */
