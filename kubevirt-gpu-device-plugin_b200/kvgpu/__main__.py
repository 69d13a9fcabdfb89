"""python -m kvgpu — InitiateDevicePlugin() of the reference (device_plugin.go:89-96, cmd/main.go) on
top of the GPU scan: createIommuDeviceMap + createVgpuIDMap through libkvgpu.so, then one
DevicePlugin server per device id / vGPU type, registered with the kubelet.

  python -m kvgpu --once --dump            scan, print the canonical dump, exit (no servers)
  python -m kvgpu --once --plugins         scan, print what each plugin would advertise (JSON)
  python -m kvgpu                          scan, serve, watch the device nodes, run until SIGTERM

There is no CPU fallback: without a usable CUDA device the scan fails and the process exits non-zero
(the reference would log the failed walk and start no plugin)."""
import argparse
import json
import signal
import sys
import threading


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m kvgpu", description=__doc__.split("\n\n")[0])
    ap.add_argument("--pci-ids", default="/usr/pci.ids", help="pciIdsFilePath (device_plugin.go:44)")
    ap.add_argument("--base-path", default="/sys/bus/pci/devices", help="basePath (:42)")
    ap.add_argument("--vgpu-base-path", default="/sys/bus/mdev/devices", help="vGpuBasePath (:43)")
    ap.add_argument("--root-path", default="/", help="rootPath for /dev/iommu and EGM discovery")
    ap.add_argument("--socket-dir", default=None, help="kubelet device-plugin directory (pluginapi.DevicePluginPath)")
    ap.add_argument("--device", type=int, default=0, help="CUDA device running the scan")
    ap.add_argument("--once", action="store_true", help="scan and print, do not serve")
    ap.add_argument("--dump", action="store_true", help="print the canonical dump of the five maps")
    ap.add_argument("--plugins", action="store_true", help="print the plugin specs as JSON")
    args = ap.parse_args(argv)

    from . import DiscoveryScan, KvgError, canonical_dump
    try:
        ds = DiscoveryScan(args.pci_ids, args.base_path, args.vgpu_base_path, args.device)
    except KvgError as e:
        print("kvgpu: cannot create the scan context (no CPU fallback): %s" % e, file=sys.stderr)
        return 2
    try:
        ds.create_iommu_device_map()      # :91
        ds.create_vgpu_id_map()           # :93
        specs = ds.create_device_plugins()
        if args.dump:
            sys.stdout.write(canonical_dump(ds.maps).decode("latin-1"))
        if args.plugins:
            json.dump([{"key": s.key, "device_name": s.device_name, "resource_name": s.resource_name,
                        "socket_path": s.socket_path, "env_key": s.env_key, "vgpu": s.vgpu, "devs": s.devs}
                       for s in specs], sys.stdout, indent=1)
            sys.stdout.write("\n")
        if args.once:
            return 0
        from . import dpapi, serve
        sockdir = args.socket_dir or dpapi.DEVICE_PLUGIN_PATH
        allocate_check = serve.AllocateCheck(ds.ctx.pci_allocate_check, args.base_path)
        vgpu_check = serve.MdevLabelCheck(ds.ctx.mdev_label_match, args.vgpu_base_path)
        prefer = serve.NumaPacker(ds.ctx.preferred_allocation)
        plugins = serve.plugins_from_specs(specs, ds.maps, None, vgpu_check=vgpu_check, prefer=prefer,
                                           allocate_check=allocate_check, socket_dir=sockdir, base_path=args.base_path, root_path=args.root_path,
                                           vgpu_base_path=args.vgpu_base_path)
        watchers, started = [], []
        for p in plugins:                 # createDevicePlugins :131-137, :158-165: a failed start is logged, the rest go on
            try:
                p.start()
                started.append(p)
                w = serve.DeviceNodeWatcher(p)   # device nodes (or mdev nodes) + the plugin socket
                w.start()
                watchers.append(w)
            except Exception as e:        # noqa: BLE001
                print("kvgpu: error starting the %s device plugin: %s" % (p.device_name, e), file=sys.stderr)
        stop = threading.Event()
        for sig in (signal.SIGTERM, signal.SIGINT):
            signal.signal(sig, lambda *_: stop.set())
        stop.wait()                        # <-stop (:166)
        for w in watchers:
            w.stop()
        for p in started:
            p.stop()
        return 0
    finally:
        ds.close()


if __name__ == "__main__":
    sys.exit(main())
