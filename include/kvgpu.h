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
 *   kvg_health_rescan_mdev                <- the vGPU health check: device-path Create / Remove / Rename and
 *                                            NVML XID critical errors, generic_vgpu_device_plugin.go:280-385
 *   kvg_health_rescan_groups              <- the passthrough health check: Create / Remove / Rename of the IOMMU
 *                                            group's VFIO node, generic_device_plugin.go:611-690
 *   kvg_health_rescan_*_keyed             <- the same two checks with the state kept per UUID / address, so it
 *                                            survives re-scans that change the device list (the reference never
 *                                            re-scans)
 *   kvg_health_rescan_*_raw               <- the same two checks from the raw reads of the advertised devices,
 *                                            state kept per entry name, groups and parents compared as strings:
 *                                            generic_device_plugin.go:611-690, generic_vgpu_device_plugin.go:280-385,
 *                                            readers device_plugin.go:202-238, :269-284
 *   kvg_scan_pci_raw                      <- createIommuDeviceMap from the raw reads of its walk callback:
 *                                            readIDFromFileFunc :294-302, readNUMANodeFunc :304-320,
 *                                            readLinkFunc :323-331, isSupportedVfioDriver :249-252
 *   kvg_scan_mdev_raw                     <- createVgpuIDMap from the raw reads of its walk callback:
 *                                            readVgpuIDFromFileFunc :334-344, readGpuIDForVgpuFunc :347-357,
 *                                            readNUMANodeFunc :304-320
 *   kvg_scan_pci_delta                   <- (no reference equivalent: the reference never re-scans)
 *   kvg_scan_mdev_delta                   <- (no reference equivalent: createVgpuIDMap runs once)
 *   kvg_scan_pci_raw_delta                <- (no reference equivalent: the reference never re-scans)
 *   kvg_scan_mdev_raw_delta               <- (no reference equivalent: the reference never re-scans)
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
  KVG_ERANGE = -6, /* output buffer too small / value does not fit the wire format */
  KVG_EPANIC = -7  /* the Go reference would panic on this input (kvg_scan_pci_raw, kvg_scan_mdev_raw) */
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
/* The reads of createIommuDeviceMap's walk callback (device_plugin.go:191-246), raw, one entry per visited
 * non-directory Walk entry in Walk order, decoded on the GPU into the records above, then scanned as kvg_scan_pci
 * scans them.  Field f of entry i is bytes[off[i*KVG_RAW_FIELDS + f] .. off[i*KVG_RAW_FIELDS + f + 1]): the entry
 * name, the vendor, device and numa_node file contents as os.ReadFile returned them, and the driver and iommu_group
 * link TARGETS as os.Readlink returned them.  state[i] bit f: read f was made; bit 8 + f: it failed (the bits of
 * KVG_RAW_NAME are unused).  A read the reference does not reach may be skipped or made: the answer is the same. */
enum { KVG_RAW_NAME, KVG_RAW_VENDOR, KVG_RAW_DRIVER, KVG_RAW_GROUP, KVG_RAW_NUMA, KVG_RAW_DEVICE, KVG_RAW_FIELDS };
typedef struct kvg_pci_raw {
  size_t n;
  const uint32_t *off;   /* [n * KVG_RAW_FIELDS + 1], off[0] == 0, non-decreasing */
  const uint8_t *bytes;  /* [off[n * KVG_RAW_FIELDS]] */
  const uint16_t *state; /* [n] */
} kvg_pci_raw;

/* The snapshot kvg_scan_pci_raw decoded (library-owned; kvg_result_free).  recs are what the host snapshotter packs:
 *   packed_addr     1: addr is the packed BDF (every name is a canonical "dddd:bb:dd.f" and they ascend strictly);
 *                   0: addr is the Walk index
 *   groups_numeric  1: iommu_group is the link basename as a number (every non-empty basename reached is a canonical
 *                   decimal below 2^32); 0: the handle of the basename, handles in order of first appearance from 0
 *                   (an entry without a group also holds 0); group h = group_bytes[group_off[h] .. group_off[h + 1])
 *   devices_numeric 1: device is the id as a number (every device string read is four lower-case hex digits);
 *                   0: the handle of the string, as for groups (at most 65,536); device names are then asked per key
 *                   through kvg_name_lookup, the result's name join is keyed by the handle and does not apply. */
typedef struct kvg_pci_snap {
  uint64_t n_records;
  const kvg_pci_rec *recs;
  uint8_t packed_addr, groups_numeric, devices_numeric;
  uint32_t n_group_names;
  const uint32_t *group_off; /* [n_group_names + 1] */
  const uint8_t *group_bytes;
  uint32_t n_device_names;
  const uint32_t *device_off; /* [n_device_names + 1] */
  const uint8_t *device_bytes;
} kvg_pci_snap;

/* Decode `raw` on the GPU with the reference's rules, in its short-circuit order (device_plugin.go:202-238):
 *   vendor       data[2:], Trim "\n" (:294-302); four lower-case hex digits give the number, anything else 0xffff;
 *                the rest is read only for "10de" (:209)
 *   driver       the link basename (:323-331), then the dictionary of isSupportedVfioDriver (:249-252)
 *   iommu_group  the link basename (:221-225)
 *   numa_node    strings.TrimSpace over UTF-8 (unicode.IsSpace; an invalid byte is not a space), then
 *                strconv.ParseInt(s, 10, 64); an error sets KVG_PF_NUMA_ERR (:226-230, :304-320); the value stays raw
 *   device       data[2:], Trim "\n" (:234-238)
 * choose the snapshot modes (kvg_pci_snap), intern the columns in index mode, pack the records into the context's
 * record staging and scan them as kvg_scan_pci does: *res equals kvg_scan_pci(ctx, (*snap)->recs, n).  The call writes
 * the scan state kvg_scan_pci writes and nothing else (delta, health and allocation state are untouched).
 * Launches: one decode; per column in index mode one probe and one compaction; one pack unless every column is
 * numeric; then the scan's.  The host waits for the decode (one synchronisation) and, in index mode, for the intern.
 * Errors (neither writes *res or *snap):
 *   KVG_EINVAL  nothing launched: ctx, raw, res or snap NULL; off or state NULL with n > 0; bytes NULL with bytes to
 *               read; off[0] != 0 or decreasing offsets; n above 0xfffffff0 (the scan's bound).  Found by the decode:
 *               a read the reference reaches was not made (kvg_last_error names the lowest entry and the file).
 *   KVG_EPANIC  the reference would panic: data[2:] of a vendor or device file shorter than 2 bytes that it reaches;
 *               kvg_last_error names the lowest such entry and the file.  Beats KVG_ERANGE.
 *   KVG_ERANGE  a reached numa_node that parses but does not fit int16, or more than 65,536 distinct device strings
 *               in index mode (the lowest entry is named).
 *   KVG_ESTATE  before kvg_pciids_load, as kvg_scan_pci; a pending parse is handled as there.
 * n = 0: an empty result and snapshot, nothing launched and no scan state changed. */
int kvg_scan_pci_raw(kvg_ctx *ctx, const kvg_pci_raw *raw, kvg_pci_result **res, kvg_pci_snap **snap);
/* The reads of createVgpuIDMap's walk callback (device_plugin.go:259-290), raw, one entry per visited non-directory
 * Walk entry of the mdev bus in Walk order, decoded on the GPU into kvg_mdev_rec records and a type dictionary, then
 * scanned as kvg_scan_mdev scans them.  The off / state conventions are those of kvg_pci_raw with KVG_MRAW_FIELDS
 * fields per entry: the entry name; the mdev_type/name contents as os.ReadFile returned them; the os.Readlink TARGET
 * of the entry itself; the numa_node contents of the parent.
 *   KVG_MRAW_NUMA is <pci base>/<P>/numa_node, where P is what readGpuIDForVgpuFunc (:347-357) returns for the
 *   KVG_MRAW_LINK target.  This path is the one thing the host derives, because it has to name the file; the record's
 *   parent key still comes from the GPU's own decode of KVG_MRAW_LINK. */
enum { KVG_MRAW_NAME, KVG_MRAW_TYPE, KVG_MRAW_LINK, KVG_MRAW_NUMA, KVG_MRAW_FIELDS };
typedef struct kvg_mdev_raw {
  size_t n;
  const uint32_t *off;   /* [n * KVG_MRAW_FIELDS + 1], off[0] == 0, non-decreasing */
  const uint8_t *bytes;  /* [off[n * KVG_MRAW_FIELDS]] */
  const uint16_t *state; /* [n] bit f: read f was made; bit 8 + f: it failed (the bits of KVG_MRAW_NAME are unused) */
} kvg_mdev_raw;

/* The snapshot kvg_scan_mdev_raw decoded (library-owned; kvg_result_free).  recs are what the host snapshotter packs:
 *   uuid_ok         1: uuid holds the name's 16 bytes (every name is a canonical lower-case 8-4-4-4-12 UUID and they
 *                   ascend strictly); 0: bytes 0..3 of uuid are the Walk index, big-endian, the rest 0
 *   parents_packed  1: parent is the packed BDF of the decoded parent (every decoded parent, an empty one included, is
 *                   a canonical "dddd:bb:dd.f"); 0: the handle of the parent string, handles in order of first
 *                   appearance from 0; parent h = parent_bytes[parent_off[h] .. parent_off[h + 1])
 *   A record without a decoded parent holds 0 either way (its record is dropped by the scan).
 *   type_idx indexes the raw type dictionary: the distinct mdev_type/name contents in order of first appearance, type
 *   h = type_bytes[type_off[h] .. type_off[h + 1]) (a record whose type read failed holds 0). */
typedef struct kvg_mdev_snap {
  uint64_t n_records;
  const kvg_mdev_rec *recs;
  uint8_t uuid_ok, parents_packed;
  uint32_t n_types;
  const uint32_t *type_off; /* [n_types + 1] */
  const uint8_t *type_bytes;
  uint32_t n_parent_names;    /* 0 when parents_packed */
  const uint32_t *parent_off; /* [n_parent_names + 1] */
  const uint8_t *parent_bytes;
} kvg_mdev_snap;

/* Decode `raw` on the GPU with the reference's rules, in its short-circuit order (device_plugin.go:269-284):
 *   mdev_type/name  a failed read sets KVG_MF_TYPE_ERR and nothing else is reached; otherwise the raw bytes (empty
 *                   included) are the type string, interned into the raw type dictionary (the label rule :341-342
 *                   stays in the scan)
 *   link            reached when the type read succeeded; a failed read sets KVG_MF_PARENT_ERR.  The parent is
 *                   strings.Split(target, "/")[len-2] with Trim "\n" (:347-357): the bytes between the second-to-last
 *                   '/' (or the start) and the last '/'; it may be empty.  No '/' at all: the reference panics.
 *   numa_node       reached when a parent was decoded: strings.TrimSpace over UTF-8, then strconv.ParseInt(s, 10, 64)
 *                   (:304-320); a failed read or a parse error sets KVG_MF_NUMA_ERR and keeps the record with 0
 * choose the snapshot modes (kvg_mdev_snap), intern the type strings (always) and the parents (index mode), pack the
 * records into the context's record staging and scan them as kvg_scan_mdev does: *res equals
 * kvg_scan_mdev(ctx, (*snap)->recs, n, &dict), where dict is the snapshot's type dictionary.  The call writes the scan
 * state kvg_scan_mdev writes and nothing else (the mdev delta, mdev health and allocation state are untouched).
 * Launches: one decode; one probe and one compaction for the types, and for the parents in index mode; one pack; then
 * the scan's.  The host waits for the decode (one synchronisation) and for the intern (one more).
 * Errors (none writes *res or *snap):
 *   KVG_EINVAL  nothing launched: ctx, raw, res or snap NULL; off or state NULL with n > 0; bytes NULL with bytes to
 *               read; off[0] != 0 or decreasing offsets; n above 0xfffffff0.  Found by the decode: a read the
 *               reference reaches was not made (kvg_last_error names the lowest entry and the file).
 *   KVG_EPANIC  the reference would panic: a reached link target without '/' (splitStr[len-2], :353); kvg_last_error
 *               names the lowest such entry.  Beats KVG_ERANGE.
 *   KVG_ERANGE  a reached numa_node that parses but does not fit int16, or a 65,536th distinct type string (the
 *               65,535-type limit of kvg_scan_mdev); the lowest entry is named.
 *   KVG_ESTATE  before kvg_pciids_load, as kvg_scan_mdev.
 * n = 0: an empty result and snapshot, nothing launched and no scan state changed. */
int kvg_scan_mdev_raw(kvg_ctx *ctx, const kvg_mdev_raw *raw, kvg_mdev_result **res, kvg_mdev_snap **snap);
/* Allocate-time re-check of the vGPU plugin (generic_vgpu_device_plugin.go:216-221): match[i] = 1 iff the label of
 * file i -- Trim(raw, "\n") then every RE2 \s+ run ([\t\n\f\r ]) -> "_" (device_plugin.go:341-342) -- equals the
 * name_len bytes at `name`, else 0.  `files` uses the layout of kvg_type_dict, one entry per file that WAS read; a
 * failed read never reaches the rule (the reference's `err != nil ||` short-circuits), so the caller skips it.
 * `match` is caller memory of files->n_types bytes.  One launch per call with n_types > 0, none for n_types = 0 or a
 * refused call.  Files of any length, up to the uint32 offsets.  The call uses buffers of its own: no scan, fetch,
 * delta or health state changes, so it may run between kvg_dev_scan_mdev and kvg_dev_scan_mdev_fetch.
 * KVG_EINVAL: ctx, files or match NULL; off or bytes NULL with n_types > 0; name NULL with name_len > 0; off[0] != 0
 * or decreasing offsets. */
int kvg_mdev_label_match(kvg_ctx *ctx, const kvg_type_dict *files, const uint8_t *name, size_t name_len,
                         uint8_t *match);
/* Allocate-time re-check of the passthrough plugin (generic_device_plugin.go:387-399) for every member of every
 * requested IOMMU group, in the order the reference visits them.  Record i passes iff KVG_PF_IOMMU_ERR is clear,
 * recs[i].iommu_group == want_group[i], KVG_PF_VENDOR_ERR is clear and recs[i].vendor == 0x10de; addr, device, driver,
 * numa and every other flag are ignored.  *first_bad = the smallest failing index, or n when all pass.
 * Handles: intern the group strings per call, one handle per distinct string, and use the same table for the link
 * just read (recs[i].iommu_group) and the group the maps hold (want_group[i]), so equal handles mean equal strings.
 * Never parse the strings as numbers: the reference compares strings, so "042" is not "42".  The vendor is 0x10de
 * iff the vendor file read back as exactly "10de" (any other value, e.g. 0xffff, fails).
 * One launch per call with n > 0, none for n = 0 (*first_bad = 0) or a refused call.  The call uses buffers of its
 * own: no scan, fetch, delta, health or name-table state changes, and it does not wait for a pci.ids parse, so it
 * may run between kvg_dev_scan_pci and kvg_dev_scan_pci_fetch.
 * KVG_EINVAL (nothing launched, *first_bad unwritten): ctx or first_bad NULL; recs or want_group NULL with n > 0;
 * n > UINT32_MAX.  It is kvg_pci_allocate_check with one request and no EGM device. */
int kvg_pci_group_check(kvg_ctx *ctx, const kvg_pci_rec *recs, const uint32_t *want_group, size_t n,
                        size_t *first_bad);
/* The passthrough plugin's Allocate decisions (generic_device_plugin.go:352-444) for every container request of one
 * AllocateRequest, in one launch: the re-check of kvg_pci_group_check and the EGM match of egmPathsForAllocatedGPUs
 * (:159-184).
 * Re-check: request r's records are recs / want_group from the end of request r-1's, reqs[r].n_members of them: every
 * member of every requested group, in the order the reference visits them.  Each is judged by kvg_pci_group_check's
 * rule.  first_bad[r] = the smallest failing position within the request, or reqs[r].n_members when every member
 * passes.  Group handles come from one intern table per call, as for kvg_pci_group_check ("042" is not "42").
 * EGM: intern the EGM devices' GPU strings first, into handles [0, n_egm_gpus), keyed by the reference's normalised
 * string (strings.ToLower(strings.TrimSpace(s))).  EGM device e lists its handles in egm_gpu[egm_off[e] ..
 * egm_off[e + 1]).  Request r's reqs[r].n_ids DevicesIDs follow those of requests 0..r-1 in `ids`, each the handle of
 * its normalised string if some EGM device lists that string, else any value >= n_egm_gpus.
 * egm_take[r * n_egm + e] = 1 iff every handle of device e is among request r's IDs, else 0; a device with an empty
 * list is taken, as the reference's loop takes it.  Duplicates on either side do not matter.  The reference mounts
 * the taken devices' paths, sorted.
 * One launch per call with n_reqs > 0 (requests with empty lists included), none for n_reqs = 0 or a refused call.
 * The call uses buffers of its own: no scan, fetch, delta, health or name-table state changes, and it does not wait
 * for a pci.ids parse.  egm_off (n_egm + 1 entries) may be NULL when n_egm = 0.
 * KVG_EINVAL (nothing launched, first_bad and egm_take unwritten): ctx NULL; reqs or first_bad NULL with n_reqs > 0;
 * recs or want_group NULL with n_recs > 0; ids NULL with n_ids > 0; egm_off NULL with n_egm > 0; egm_gpu NULL with a
 * non-empty list; egm_take NULL with n_reqs * n_egm > 0; member or ID counts that do not add up to n_recs / n_ids;
 * n_recs or n_ids > UINT32_MAX; egm_off[0] != 0 or decreasing offsets; an egm_gpu value >= n_egm_gpus;
 * n_egm_gpus > KVG_ALLOC_MAX_EGM_GPUS. */
#define KVG_ALLOC_MAX_EGM_GPUS 65536 /* distinct EGM GPU strings per call: one bit each in shared memory (8 KiB) */
typedef struct kvg_alloc_req {
  uint32_t n_members; /* records of this request: every member of every requested group, in the reference's order */
  uint32_t n_ids;     /* this request's DevicesIDs, as EGM handles */
} kvg_alloc_req;
int kvg_pci_allocate_check(kvg_ctx *ctx, const kvg_alloc_req *reqs, uint32_t n_reqs, const kvg_pci_rec *recs,
                           const uint32_t *want_group, size_t n_recs, const uint32_t *ids, size_t n_ids,
                           const uint32_t *egm_off, const uint32_t *egm_gpu, uint32_t n_egm, uint32_t n_egm_gpus,
                           uint32_t *first_bad, uint8_t *egm_take);
/* The passthrough plugin's Allocate decisions (generic_device_plugin.go:352-444) for every container request of one
 * AllocateRequest, decided on the GPU from the raw reads the reference makes for them: the group re-check of every
 * member (:387-399), EGM discovery's decoding of the class entries (discoverEGMDevicesFunc :120-157) and the EGM match
 * (egmPathsForAllocatedGPUs :159-184).  The host lists directories, stats and reads; it decodes nothing.
 * Members: every member of every requested group, request after request, reqs[r].n_members per request, in the order
 * the reference visits them.  Field f of member i is member_bytes[member_off[3i + f] .. member_off[3i + f + 1]):
 *   KVG_AMEM_LINK    the iommu_group link TARGET as os.Readlink returned it
 *   KVG_AMEM_VENDOR  the vendor file contents as os.ReadFile returned them
 *   KVG_AMEM_GROUP   the group string the maps hold for the member (bdfToIommu[bdf]); always present
 * member_state[i] bit f: read f was made; bit 8 + f: it failed (only LINK and VENDOR have bits).
 * IDs: the requests' DevicesIDs, reqs[r].n_ids per request; ID k = id_bytes[id_off[k] .. id_off[k + 1]).
 * EGM class entries: every entry of the EGM class directory in ReadDir order; field f of entry e is
 * egm_bytes[egm_off[2e + f] .. egm_off[2e + f + 1]): KVG_AEGM_NAME the entry name, KVG_AEGM_GPUS the gpu_devices
 * contents.  egm_state[e] bit f / 8 + f: read f made / failed, for KVG_AEGM_GPUS and for KVG_AEGM_STAT, the Stat of
 * /dev/<name> (it has no bytes).  Every offset table starts at 0 and does not decrease.
 * Rules, in the reference's short-circuit order:
 *   member     the link's basename (filepath.Split) must equal the group string byte for byte ("042" is not "42"),
 *              else the member fails and its vendor is not reached; a failed read fails it.  Then the vendor: a failed
 *              read fails the member; fewer than 2 bytes is the reference's panic (data[2:]); else Trim(data[2:], "\n")
 *              must be exactly "10de".
 *   request    first_bad[r] = the smallest failing position within the request, or reqs[r].n_members; panic[r] = 1
 *              iff the member at first_bad[r] failed by that panic (a per-request output, not a call error: an earlier
 *              request may fail first).  The reads of a request up to and including its first failing member are
 *              reached; the later ones may be made or skipped.
 *   EGM entry  egm_kept[e] = 1 iff its name has the prefix "egm", its gpu_devices read succeeded, strings.Fields of
 *              the contents (unicode.IsSpace over UTF-8; an invalid byte is RuneError, not a space) is not empty, and
 *              the Stat succeeded.  gpu_devices is reached for "egm" names, the Stat when there are fields.
 *   keys       strings.ToLower(strings.TrimSpace(s)) with Go's semantics: runes through unicode.ToLower (simple case
 *              mapping, Unicode 15.0.0), each invalid byte one U+FFFD, so "\xff" and "\xfe" are the same key.
 *              egm_take[r * n_egm + e] = 1 iff entry e is kept and the key of every field of e is the key of one of
 *              request r's IDs.  Duplicates do not matter.  The reference mounts /dev/<name> of the taken entries,
 *              sorted.
 * Launches: one member decode when there are members, one key kernel when n_egm > 0, and k_pci_allocate_check when
 * n_reqs > 0, so at most three; none for a call with no requests and no EGM entries, or one refused before launch
 * (the KVG_EINVAL argument errors below).  A refusal found on the device launches what the call would have launched.
 * One host synchronisation per call that launches.  The call uses buffers of its own: no scan, fetch, delta, health or
 * name-table state changes, and it does not wait for a pci.ids parse.
 * Errors (the outputs stay unwritten):
 *   KVG_EINVAL  nothing launched: ctx NULL; reqs, first_bad or panic NULL with n_reqs > 0; raw NULL; an offset table,
 *               state or bytes NULL with entries or bytes to read; egm_kept NULL with n_egm > 0; egm_take NULL with
 *               n_reqs * n_egm > 0; member or ID counts that do not add up; n_members or n_ids > UINT32_MAX; an offset
 *               table that does not start at 0 or decreases.  Found on the device: a reached read that was not made;
 *               kvg_last_error names the lowest (the EGM entries first, as the reference discovers them before it reads
 *               any member, then request by request).
 *   KVG_ERANGE  more than KVG_ALLOC_RAW_MAX_EGM_KEYS distinct keys among the kept entries' fields; kvg_last_error
 *               names the lowest entry that carries one beyond the cap.  A missing read beats it. */
enum { KVG_AMEM_LINK, KVG_AMEM_VENDOR, KVG_AMEM_GROUP, KVG_AMEM_FIELDS };
enum { KVG_AEGM_NAME, KVG_AEGM_GPUS, KVG_AEGM_FIELDS, KVG_AEGM_STAT = KVG_AEGM_FIELDS };
/* distinct EGM keys per call: the bitmap of kvg_pci_allocate_check, less one handle that marks an entry not kept */
#define KVG_ALLOC_RAW_MAX_EGM_KEYS (KVG_ALLOC_MAX_EGM_GPUS - 1)
typedef struct kvg_alloc_raw {
  size_t n_members;
  const uint32_t *member_off;   /* [n_members * KVG_AMEM_FIELDS + 1] */
  const uint8_t *member_bytes;
  const uint16_t *member_state; /* [n_members] */
  size_t n_ids;
  const uint32_t *id_off;       /* [n_ids + 1] */
  const uint8_t *id_bytes;
  uint32_t n_egm;
  const uint32_t *egm_off;      /* [n_egm * KVG_AEGM_FIELDS + 1] */
  const uint8_t *egm_bytes;
  const uint16_t *egm_state;    /* [n_egm] */
} kvg_alloc_raw;
int kvg_pci_allocate_raw(kvg_ctx *ctx, const kvg_alloc_req *reqs, uint32_t n_reqs, const kvg_alloc_raw *raw,
                         uint32_t *first_bad, uint8_t *panic, uint8_t *egm_kept, uint8_t *egm_take);
/* The passthrough plugin's AllocateResponse (generic_device_plugin.go:352-444) for every container request of one
 * AllocateRequest, from the raw reads: kvg_pci_allocate_raw's decisions, then readVFIODev (:702-716) of every member,
 * requestedDeviceFound, the device specs and the env value.  The host plans (bdfToIommu / iommuMap lookups), lists,
 * reads and stats; it decides nothing.  `reqs` and `raw` are kvg_pci_allocate_raw's, with request r's members those of
 * its visited IDs, ID after ID, each ID's group members in map order.
 * Plan: request r visits its first in->n_visited[r] DevicesIDs; in->lookup_error[r] = 1 when its next ID misses
 * bdfToIommu or has an empty iommuMap entry.  in->id_members[v] is the member count of visited ID v (request after
 * request); the counts of request r add up to reqs[r].n_members.
 * Members: addr_bytes[addr_off[i] .. addr_off[i + 1]) is dev.addr as the maps hold it.  The vfio-dev listing of member
 * i is entries vfio_first[i] .. vfio_first[i + 1], in any order: name vfio_bytes[vfio_off[e] .. vfio_off[e + 1]) and
 * vfio_dir[e] = DirEntry.IsDir() (a link is not a directory).  vfio_state[i]: KVG_AVFIO_MADE when the listing was
 * made, | KVG_AVFIO_FAILED when os.ReadDir failed (the host keeps the OS error text).  It is reached when iommufd = 1
 * (supportsIOMMUFD; its other errors are raised by the host before the call) and the member passed the re-check.
 * Rules, per request in the reference's order (visited ID k, then its members):
 *   member    the re-check of kvg_pci_allocate_raw fails it: UNKNOWN_MEMBER, or PANIC for the vendor read's panic;
 *             then, with iommufd, readVFIODev: a failed listing is VFIO_READ; else the byte-wise least name with the
 *             prefix "vfio" among the entries that are directories, none being VFIO_NONE ("no iommufd device found")
 *   ID        after its members: no member whose dev.addr equals the ID byte for byte is UNKNOWN_ID
 *   request   after the visited IDs: lookup_error is UNKNOWN_ID at n_visited
 *   specs     per visited ID: /dev/vfio/devices/<name> per member (iommufd), /dev/vfio/vfio,
 *             filepath.Join("/dev/vfio", group) ("" and "." give /dev/vfio, ".." gives /dev), /dev/iommu (iommufd);
 *             then /dev/<name> of the EGM entries the request takes (kvg_pci_allocate_raw's rule), ascending.  A host
 *             path is kept at its first occurrence (appendDeviceSpec); container path = host path, permissions "mrw".
 *   env       envList outlives the request loop (:361): response r's value is the addresses of every member of
 *             requests 0..r joined by ',' (duplicates kept), a prefix of env_bytes of env_len[r] bytes; env_key[r] = 1
 *             iff requests 0..r visited an ID (else envs is empty).
 * Requests are decided independently; the caller returns the error of the first request whose error is not OK.
 * error_at[r]: the ID index within the request for UNKNOWN_ID, the member position within the request for the
 * other errors, 0 for OK.
 * Output: *res, library-owned (kvg_result_free).  Request r's specs are spec_span[2s] (offset into spec_bytes) and
 * spec_span[2s + 1] (length) for s in spec_first[r] .. spec_first[r] + n_specs[r]; an erring request has none.
 * Launches: k_araw_members when there are members; k_aresp_members when there are members or two EGM entries;
 * k_araw_keys when there are EGM entries; k_pci_allocate_check and k_aresp_requests when there are requests, so at
 * most five, none for a call with no requests and no EGM entries (*res is an empty result) or one refused before
 * launch.  One host synchronisation per call that launches; the outputs land in mapped host memory sized on the host
 * from the inputs.  The call uses buffers of its own: no scan, fetch, delta, health or name-table state changes, and
 * it does not wait for a pci.ids parse.
 * Errors (*res unwritten):
 *   KVG_EINVAL  before launch: every argument refusal of kvg_pci_allocate_raw; in or res NULL; a plan or listing table
 *               NULL with entries; vfio_first or vfio_off not starting at 0 or decreasing; visit counts that do not
 *               add up; n_visited + lookup_error > n_ids; a visited ID with no members.  Found on the device, in this
 *               order: members of one visited ID with different group strings, or a group string holding '/'; EGM
 *               entry names that do not ascend strictly byte-wise; then kvg_pci_allocate_raw's refusals in its order,
 *               a reached listing that was not made taking its place beside a request's missing member read
 *               (kvg_last_error names the entry).
 *   KVG_ERANGE  kvg_pci_allocate_raw's key cap; a response of more than 2^32 - 1 spec slots or pool bytes. */
enum { KVG_ARESP_OK, KVG_ARESP_UNKNOWN_ID, KVG_ARESP_UNKNOWN_MEMBER, KVG_ARESP_PANIC, KVG_ARESP_VFIO_READ,
       KVG_ARESP_VFIO_NONE };
enum { KVG_AVFIO_MADE = 1, KVG_AVFIO_FAILED = 2 };
typedef struct kvg_alloc_resp_in {
  uint32_t iommufd;             /* supportsIOMMUFD: 0 or 1 */
  const uint32_t *n_visited;    /* [n_reqs] */
  const uint8_t *lookup_error;  /* [n_reqs] */
  const uint32_t *id_members;   /* [sum of n_visited] */
  const uint32_t *addr_off;     /* [n_members + 1] */
  const uint8_t *addr_bytes;
  const uint32_t *vfio_first;   /* [n_members + 1] */
  const uint32_t *vfio_off;     /* [vfio_first[n_members] + 1] */
  const uint8_t *vfio_bytes;
  const uint8_t *vfio_dir;      /* [vfio_first[n_members]] */
  const uint8_t *vfio_state;    /* [n_members] */
} kvg_alloc_resp_in;
typedef struct kvg_alloc_resp {
  uint32_t n_reqs;
  const uint8_t *error;         /* [n_reqs] KVG_ARESP_* */
  const uint32_t *error_at;     /* [n_reqs] */
  const uint32_t *spec_first;   /* [n_reqs] */
  const uint32_t *n_specs;      /* [n_reqs] */
  const uint32_t *spec_span;    /* [2 * spec slots] */
  const uint8_t *spec_bytes;
  const uint32_t *env_len;      /* [n_reqs] */
  const uint8_t *env_key;       /* [n_reqs] */
  const uint8_t *env_bytes;
} kvg_alloc_resp;
int kvg_pci_allocate_response(kvg_ctx *ctx, const kvg_alloc_req *reqs, uint32_t n_reqs, const kvg_alloc_raw *raw,
                              const kvg_alloc_resp_in *in, kvg_alloc_resp **res);
/* GetPreferredAllocation of the passthrough plugin (generic_device_plugin.go:470-608): the NUMA packing of every
 * container request of one PreferredAllocationRequest, in one launch.
 * Entries: request r's entries follow those of requests 0..r-1 in `ids`, its n_must must-include IDs first, then its
 * n_avail available IDs, each list in kubelet order (duplicates and IDs the plugin does not know included).
 * Interning, per request: handle = one index per distinct ID string (< n_must + n_avail), so equal handles mean equal
 * strings; node = one index per distinct NUMA node value (< n_must + n_avail), or KVG_PREF_NODE_NONE for an ID that
 * is not a device of the plugin, a device without topology, or a device whose node is -1.  Equal handles carry equal
 * nodes.  The device's node is that of its last entry in the plugin's device list that has topology.  Nodes are only
 * compared for equality, so any other value (e.g. -2) is an ordinary node.
 * Rule, with P = the number of distinct must-include IDs: P > size (size may be 0 or negative) fails with
 * res[r].n_out = -1.  Otherwise the picks are the must-include IDs in order, then -- when P < size -- the IDs of the
 * first candidate node (must-include nodes in order of first appearance, then the nodes of `available` in order of
 * first appearance) whose must-include IDs plus available entries of other IDs (duplicates counted) reach size,
 * unless that node is KVG_PREF_NODE_NONE, then available IDs in order until size; an ID is never picked twice.
 * Output: res[r] = {n_out, P}; out_pos[first entry of r ..] holds r's n_out picks as entry positions within r
 * (0 = its first must-include entry), in the order the reference appends them.  out_pos has room for n_ids positions;
 * a failed request writes none.  The reference's error text is
 * "number of MustIncludeDeviceIDs (P) exceeds allocation size (size)" for the first failing request.
 * One launch per call with n_reqs > 0 (requests with empty lists included: they still take the size test), none for
 * n_reqs = 0 or a refused call.  The call uses buffers of its own: no scan, fetch, delta, health or name-table state
 * changes, and it does not wait for a pci.ids parse.
 * KVG_EINVAL (nothing launched, res unwritten): ctx NULL; reqs or res NULL with n_reqs > 0; ids or out_pos NULL with
 * n_ids > 0; n_ids > UINT32_MAX; sum of n_must + n_avail != n_ids; a handle or node out of its request's range. */
#define KVG_PREF_NODE_NONE 0xffffffffu /* the reference's -1: no topology, node -1, or not a device of the plugin */
typedef struct kvg_pref_id {
  uint32_t handle, node;
} kvg_pref_id;
typedef struct kvg_pref_req {
  uint32_t n_must, n_avail;
  int32_t size; /* allocation_size */
  uint32_t pad;
} kvg_pref_req;
typedef struct kvg_pref_res {
  int32_t n_out; /* -1: more distinct must-include IDs than size */
  uint32_t n_must_distinct;
} kvg_pref_res;
int kvg_preferred_allocation(kvg_ctx *ctx, const kvg_pref_req *reqs, uint32_t n_reqs, const kvg_pref_id *ids,
                             size_t n_ids, kvg_pref_res *res, uint32_t *out_pos);
/* Classify `recs`, diff against the alive-set of the previous call on this context (first call:
 * against "nothing alive").  A call with a different n re-arms the same way, as does
 * kvg_health_reset(); n = 0 returns an empty delta.  Pinned (cudaHostAlloc / registered) `recs` of
 * at most 32,768 records are read in place by TMA bulk copies and must be 16-byte aligned; this is
 * not checked.  Pageable memory is staged and has no alignment requirement. */
int kvg_health_rescan(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n, kvg_health_delta **delta);
int kvg_health_reset(kvg_ctx *ctx);

/* Health re-scan of mdev records: a vGPU is healthy while its record is present (createVgpuIDMap's keep rule) and not
 * marked by a critical XID on its parent GPU.
 *
 * `xid_parents` holds the parent handles (kvg_mdev_rec.parent) of the GPUs that reported an XID since the previous
 * call: a one-shot list of events, not a standing set.  Order and duplicates do not matter; membership is exact
 * uint32 equality, so a handle no record carries marks nothing.  Record i keeps two bits from the previous call, p
 * (present) and m (marked), m implies p:
 *
 *   p' = record i passes createVgpuIDMap's keep rule with n_types dictionary entries
 *   m' = p' && (parent(i) in xid_parents || (p && m))
 *   healthy before h = p && !m, healthy now h' = p' && !m'; i is listed iff h' != h
 *
 * So a mark stays until the record vanishes; a vGPU that comes back is healthy unless its parent is in xid_parents on
 * that same call (generic_vgpu_device_plugin.go:330-351: only a Create sends `healthy`).  The delta is
 * kvg_health_delta: n_alive counts the records healthy now, changed[] holds (index << 1) | healthy_now in ascending
 * index order.
 *
 * A call with a different n re-arms the state to "nothing present, nothing marked", as does kvg_health_mdev_reset();
 * n = 0 returns an empty delta.  n_xid > KVG_HEALTH_MAX_XID, or xid_parents == NULL with n_xid > 0, returns
 * KVG_EINVAL and leaves the state unchanged.  The state is the context's own, separate from kvg_health_rescan's:
 * kvg_health_rescan, kvg_health_reset, every scan, every delta and kvg_pciids_load leave it unchanged, and this call
 * leaves theirs unchanged.
 *
 * Up to 32,768 records and with kernel timing off, the call is one kernel launch with no driver synchronisation on the
 * way back; pinned `recs` are then read in place and must be 16-byte aligned (not checked).  Pageable memory is staged
 * and has no alignment requirement. */
#define KVG_HEALTH_MAX_XID 1024 /* parent handles per call */
int kvg_health_rescan_mdev(kvg_ctx *ctx, const kvg_mdev_rec *recs, size_t n, uint32_t n_types,
                           const uint32_t *xid_parents, size_t n_xid, kvg_health_delta **delta);
int kvg_health_mdev_reset(kvg_ctx *ctx);

/* Health re-scan of PCI records by IOMMU group: a passthrough GPU is healthy while its record passes
 * createIommuDeviceMap's filter and the VFIO node of its IOMMU group (/dev/vfio/<group>) exists.
 *
 * `group_nodes` holds the handles of the IOMMU groups whose device node exists now, in the encoding of
 * kvg_pci_rec.iommu_group: a standing set (one listing of the VFIO device directory per tick), not a list of events.
 * Order and duplicates do not matter; membership is exact uint32 equality, so a handle no record carries changes
 * nothing.  Record i keeps one bit h from the previous call:
 *
 *   h' = record i passes createIommuDeviceMap's filter (as kvg_health_rescan) && iommu_group(i) in group_nodes
 *   i is listed iff h' != h
 *
 * So when every group of the snapshot has a node, the call reports what kvg_health_rescan reports on the same
 * sequence of snapshots; and when every record passes the filter, all devices of a group flip together, exactly when
 * the group's node appears or vanishes (generic_device_plugin.go:611-690: a Create sends `healthy`, a Remove or Rename
 * `unhealthy`, for every device of the group).  The delta is kvg_health_delta: n_alive counts the records healthy now,
 * changed[] holds (index << 1) | healthy_now in ascending index order.
 *
 * A call with a different n re-arms the state to "nothing healthy", as does kvg_health_groups_reset(); n = 0 returns
 * an empty delta.  n_nodes > KVG_HEALTH_MAX_GROUPS, or group_nodes == NULL with n_nodes > 0, returns KVG_EINVAL and
 * leaves the state unchanged.  The state is the context's own, separate from those of kvg_health_rescan and
 * kvg_health_rescan_mdev: those calls, their resets, every scan, every delta and kvg_pciids_load leave it unchanged,
 * and this call leaves theirs unchanged.
 *
 * Up to 32,768 records and with kernel timing off, the call is one kernel launch with no driver synchronisation on the
 * way back; pinned `recs` are then read in place and must be 16-byte aligned (not checked).  Pageable memory is staged
 * and has no alignment requirement. */
#define KVG_HEALTH_MAX_GROUPS 4096 /* group handles per call */
int kvg_health_rescan_groups(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n, const uint32_t *group_nodes,
                             size_t n_nodes, kvg_health_delta **delta);
int kvg_health_groups_reset(kvg_ctx *ctx);

/* Keyed health re-scans: kvg_health_rescan_mdev and kvg_health_rescan_groups with the state kept per device KEY
 * instead of per record index, so a device keeps its state while the list of records around it changes (a vGPU
 * created on another GPU does not clear the XID marks of the vGPUs already listed).
 *
 * Key: for mdev records the UUID, compared as 16 big-endian bytes (the order of kvg_scan_mdev_delta); for PCI records
 * kvg_pci_rec.addr as a uint32.  Within one call the keys must ascend strictly.
 *
 * State: each kind keeps a list of (key, state byte) in ascending key order, empty at first.  It is separate from the
 * index-keyed states and from every scan and delta: none of those calls or their resets touch it, and these calls
 * touch none of theirs.  For each record i of a call, with key k_i:
 *
 *   prior_i = the state byte of k_i in the previous list, or 0 if k_i is absent from it
 *   s_i     = the next state of the index-keyed rule from record i and prior_i (kvg_health_rescan_mdev with the XID
 *             parents xid_parents; kvg_health_rescan_groups with the standing node set group_nodes)
 *   record i is listed iff bit 0 (healthy) of s_i and prior_i differ
 *
 * The list then becomes {(k_i, s_i)}: keys missing from this call are forgotten.  So a vGPU keeps its XID mark while
 * it stays in the list and present; one that leaves the list and returns later starts unmarked.  When every call
 * carries the same key list, each delta is byte for byte that of the index-keyed call from a fresh state.
 *
 * The delta is kvg_health_delta: changed[] holds (i << 1) | healthy_now, i a position in THIS call's records,
 * ascending; n_alive counts the records healthy now.  n = 0 empties the list and returns an empty delta (the reset).
 *
 * Refused with KVG_EINVAL, the list unchanged and nothing handed out: keys not strictly ascending (found on the device;
 * text in kvg_last_error), n_xid > KVG_HEALTH_MAX_XID or n_nodes > KVG_HEALTH_MAX_GROUPS, a NULL set with a non-zero
 * count.
 *
 * Cost as the index-keyed calls: up to 32,768 records and with kernel timing off, one kernel launch with no driver
 * synchronisation, pinned `recs` read in place (16-byte aligned, not checked); above that the look-back form. */
int kvg_health_rescan_mdev_keyed(kvg_ctx *ctx, const kvg_mdev_rec *recs, size_t n, uint32_t n_types,
                                 const uint32_t *xid_parents, size_t n_xid, kvg_health_delta **delta);
int kvg_health_rescan_groups_keyed(kvg_ctx *ctx, const kvg_pci_rec *recs, size_t n,
                                   const uint32_t *group_nodes, size_t n_nodes, kvg_health_delta **delta);

/* Health re-scans from raw reads: the two checks of the keyed calls (generic_device_plugin.go:611-690,
 * generic_vgpu_device_plugin.go:280-385) on the raw reads of the advertised devices, decoded on the GPU by the
 * decoders of kvg_scan_pci_raw / kvg_scan_mdev_raw (the readers of device_plugin.go:202-238 and :269-284), with the
 * state kept per ENTRY NAME and every identity compared as bytes, so nothing is interned on the host.
 *
 * Entries: one per advertised device, in the kvg_pci_raw / kvg_mdev_raw layout and with its conventions (offsets,
 * the made / failed bits, a read the reference does not reach may be made or skipped).  The entry name
 * (KVG_RAW_NAME / KVG_MRAW_NAME) is the device's ID as advertised, in any form; names must ascend strictly byte-wise
 * across all entries, alive or not (checked on the device).
 *
 * Sets: `nodes` and `xid_parents` use the layout of kvg_type_dict as a list of byte strings (NULL = empty list), in
 * any order, duplicates allowed.  `nodes` is one raw listing of the VFIO device directory (a standing set);
 * `xid_parents` holds the bus ids of the GPUs that reported a critical XID since the previous call (events).
 *
 * Rules, for entry i decoded as the raw scans decode it:
 *   groups  h' = the record passes createIommuDeviceMap's filter && the iommu_group link basename equals one of the
 *           node names byte for byte ("042" is not "42"; `vfio` or `devices` match only a group so named; an empty
 *           listing means no node exists): kvg_health_rescan_groups with string membership
 *   mdev    p' = the mdev_type/name and link reads succeeded; m' = p' && (the decoded parent,
 *           Split(target, "/")[len-2] trimmed, equals one of the XID bus ids || (p && m)); an empty parent is marked by
 *           nothing.  healthy = p && !m: the two-bit rule of kvg_health_rescan_mdev
 *
 * State: each kind keeps a list of (name, state byte), byte-wise ascending.  prior_i = the byte of entry i's name in
 * the previous list, or 0; record i is listed iff bit 0 of its new byte and of prior_i differ; the list then becomes
 * this call's names and bytes.  The previous names stay on the device (double-buffered, adopted only on success).
 * Each kind has a slot of its own: no scan, delta, Allocate, kvg_pciids_load or other health call (nor its reset)
 * touches it, and these calls touch none of theirs.  A refused call hands out nothing and leaves the list unchanged.
 *
 * The delta is kvg_health_delta: changed[] holds (i << 1) | healthy_now in ascending i; n_alive counts the entries
 * healthy now.  n = 0 empties the list and returns an empty delta (the reset), with nothing launched.
 *
 * Refused, in this precedence:
 *   KVG_EINVAL  nothing launched: ctx, raw or delta NULL; off or state NULL with n > 0; bytes NULL with bytes to read;
 *               off[0] != 0 or decreasing offsets; n above 2^31 - 1; more than KVG_HEALTH_MAX_GROUPS node names or
 *               KVG_HEALTH_MAX_XID bus ids; a set with n_types > 0 and off NULL (or bytes NULL with bytes), off[0] != 0
 *               or decreasing offsets; the entries' and the set's bytes together above 4 GiB.  No byte cap applies to
 *               the set: the per-CTA table holds hashes and indices, the strings stay in device memory.
 *   KVG_EINVAL  found by the decode: a read the reference reaches was not made (kvg_last_error names the entry)
 *   KVG_EPANIC  the reference would panic (data[2:] of a short vendor / device file; a link target without '/')
 *   KVG_ERANGE  a reached numa_node that parses but does not fit int16
 *   KVG_EINVAL  the names do not ascend strictly byte-wise
 *
 * Cost: the raw bytes, offsets, states and the set are staged in one host-to-device copy.  Up to 32,768 entries and
 * with kernel timing off, one kernel launch (one CTA: the set table, the decode, the join by name and the transition
 * list written into mapped host memory) and one host synchronisation (a flag in that memory).  Above that, one launch
 * of the look-back form (k_compact over 2048-entry tiles, one set table per CTA), one copy of the counters and the
 * verdicts with one synchronisation, and one copy of the list with another. */
int kvg_health_rescan_groups_raw(kvg_ctx *ctx, const kvg_pci_raw *raw, const kvg_type_dict *nodes,
                                 kvg_health_delta **delta);
int kvg_health_rescan_mdev_raw(kvg_ctx *ctx, const kvg_mdev_raw *raw, const kvg_type_dict *xid_parents,
                               kvg_health_delta **delta);

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

/* kvg_scan_pci_raw on `raw`, and the keyed diff of its result against the previous one, keyed by ENTRY NAME (the
 * KVG_RAW_NAME bytes), so that it is exact in every snapshot mode.
 *
 * *res and *snap are byte for byte what kvg_scan_pci_raw(ctx, raw, ...) returns, with the same errors and refusals;
 * *res, *snap and *delta are all freed with kvg_result_free.
 *
 * "Previous" is the result and snapshot of the last SUCCESSFUL kvg_scan_pci_raw_delta on this context since
 * kvg_ctx_create or kvg_scan_pci_raw_delta_reset; before any such call it is empty (and numeric).  The library keeps
 * its own copy, strings included, in a slot no other call touches: kvg_scan_pci_delta, the sharded deltas, the raw
 * scans, the health calls, the Allocate calls, kvg_pciids_load and every other reset leave it unchanged, and this
 * call changes no other delta's.  A refused call hands out nothing and leaves the previous result as it was.
 *
 * Identity: a survivor is its entry name.  Survivor names must ascend strictly byte-wise (Walk order does); this is
 * checked on the device, and a violation returns KVG_EINVAL with text in kvg_last_error, state unchanged.
 * kvg_scan_pci_raw accepts such input, but a delta is undefined without an order.
 *
 * changes: one per name that survives on exactly one side, or on both with another iommu_group string
 * (KVG_CH_GROUP), another device string (KVG_CH_DEVICE) or another clamped NUMA node (KVG_CH_NUMA), ascending by
 * name.  Strings are compared as strings: "042" is not "42", and "1db6" then "1DB6" is a change.
 *   addr                 this snapshot's address handle when the name survives now, else the previous snapshot's
 *   prev_* / now_*       each side in its own snapshot's encoding: the number in numeric mode, else a handle into
 *                        that snapshot's string table; 0 on the absent side
 *   now_index/prev_index as in kvg_scan_pci_delta
 * dev_dirty / grp_dirty: deviceMap (iommuMap) key k, indexing res->dev_keys (res->grp_keys), is dirty iff the
 * (entry name, clamped NUMA) sequence of its members, in Walk order, differs between the two results, keys being
 * matched by string; new keys are dirty.  dev_gone / grp_gone: the previous result's keys whose string has no
 * survivor now, in the previous snapshot's encoding, ascending.  The caller names a removed entry or a gone key
 * through the previous kvg_pci_snap, so it keeps that snapshot until the next call returns.
 *
 * Both snapshots fully numeric (packed_addr, groups_numeric and devices_numeric on both sides): *delta is byte for
 * byte what kvg_scan_pci_delta(snap->recs) returns for the same pair, from the same two kernels on the decoded
 * records.
 *
 * Cost beyond kvg_scan_pci_raw on the same input: numeric pair, the two launches of kvg_scan_pci_delta
 * (delta_merge, delta_lists) and one synchronisation; any other mode pair adds two re-key launches (raw_rekey: name
 * ranks, key indices and the new keys' string table; raw_xlate: each previous key to the new key with its string).
 * A snapshot with a column in index mode also has its staged walk copied, device to device, into the slot (the next
 * call's re-key reads its strings); a fully numeric one copies nothing beyond the survivors and keys. */
int kvg_scan_pci_raw_delta(kvg_ctx *ctx, const kvg_pci_raw *raw, kvg_pci_result **res, kvg_pci_snap **snap,
                           kvg_pci_delta **delta);
/* forget the previous result: the next kvg_scan_pci_raw_delta reports everything as added */
int kvg_scan_pci_raw_delta_reset(kvg_ctx *ctx);

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

/* kvg_scan_mdev_raw on `raw`, and the keyed diff of its result against the previous one, keyed by ENTRY NAME (the
 * KVG_MRAW_NAME bytes, the UUID string), so that it is exact in every snapshot mode.  The contract is that of
 * kvg_scan_pci_raw_delta with these differences:
 *   - *res and *snap are byte for byte what kvg_scan_mdev_raw returns; its slot is its own (kvg_scan_mdev_delta, the
 *     sharded deltas, the raw scans, the health calls, the Allocate calls and kvg_scan_pci_raw_delta leave it alone).
 *   - changes: one per name that survives on one side only, or on both with another sanitised type label
 *     (KVG_CH_TYPE, as kvg_scan_mdev_delta compares it), another decoded parent string (KVG_CH_PARENT) or another
 *     clamped NUMA node, ascending by name.  uuid is the record's uuid bytes from the side the handle comes from (this
 *     snapshot when the name survives now); prev_parent / now_parent are each side's own encoding (packed BDF or a
 *     handle into that snapshot's parent table); prev_type / now_type are canonical ids of each side's dictionary.
 *   - type_dirty / type_gone keep their meaning (by label).  par_dirty: gpuVgpuMap key k, indexing res->par_keys, is
 *     dirty iff the entry-name sequence of its members changed, parents matched by string; par_gone lists previous
 *     parent keys whose string has no survivor now, in the previous snapshot's encoding, ascending.
 *   - Both snapshots fully numeric (uuid_ok and parents_packed on both sides): *delta is byte for byte what
 *     kvg_scan_mdev_delta(snap->recs, dict) returns for the same pair.
 *   - Survivor names must ascend strictly byte-wise (checked on the device: KVG_EINVAL, state unchanged).
 * Cost beyond kvg_scan_mdev_raw: numeric pair, the three launches of kvg_scan_mdev_delta (mdev_delta_types,
 * mdev_delta_merge, mdev_delta_lists) and one synchronisation; any other mode pair adds the two re-key launches
 * (raw_rekey, raw_xlate). */
int kvg_scan_mdev_raw_delta(kvg_ctx *ctx, const kvg_mdev_raw *raw, kvg_mdev_result **res, kvg_mdev_snap **snap,
                            kvg_mdev_delta **delta);
/* forget the previous result: the next kvg_scan_mdev_raw_delta reports everything as added */
int kvg_scan_mdev_raw_delta_reset(kvg_ctx *ctx);

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
