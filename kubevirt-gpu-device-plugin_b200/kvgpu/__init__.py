"""kvgpu — H100-native discovery-and-classification scan for the KubeVirt GPU device plugin.

The compute lives in libkvgpu.so (hand-written sm_90a CUDA, C-ABI in include/kvgpu.h); this
package is the host-side mirror of the reference's plugin interface for that path.
"""
from ._lib import (KVG_NO_NAME, MDEV_CHANGE, MDEV_REC, MDEV_SURV, PCI_CHANGE, PCI_REC, PCI_SURV, KvgError, declared_symbols,
                   load)
from .context import Context, HealthDelta, MdevDelta, MdevResult, MdevShardResult, PciDelta, PciResult, PciShardResult
from .plugin import (DiscoveryScan, Maps, MdevMapsTouched, MdevSnapshot, NvidiaGpuDevice, PciMapsTouched, PciSnapshot, PluginSpec,
                     ReferencePanic, apply_mdev_delta, apply_pci_delta, canonical_dump, format_bdf, format_uuid,
                     mdev_maps_from_result, parse_bdf, pci_maps_from_result, plugin_specs_from_maps,
                     snapshot_mdev_tree,
                     snapshot_pci_tree)
from .parallel import (MdevShardDelta, PciShardDelta, ShardedScan, allgatherv_torch, apply_mdev_shard_delta,
                       apply_pci_shard_delta, concat_in_rank_order, mdev_maps_from_shard, mdev_shard_delta_part,
                       merge_mdev_shard_deltas, merge_parts, merge_pci_shard_deltas, pci_maps_from_shard,
                       shard_delta_part, shard_range)

__all__ = [n for n in dir() if not n.startswith("_")]
