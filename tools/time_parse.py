"""Parse (K1) timing at 256 images (scan kernel GB/s, family times) and at a single image."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "kubevirt-gpu-device-plugin_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np, torch, kvgpu
import bench as B
text = B.load_pciids()
ctx = kvgpu.Context(0)
pad = ctx.text_pad(len(text))
h = np.full(pad + 16, 10, dtype=np.uint8); h[:len(text)] = np.frombuffer(text, dtype=np.uint8)
d = torch.from_numpy(h).cuda()
nf = 256; stride = pad + 16
big = d[:stride].repeat(nf); torch.cuda.synchronize()
for _ in range(3): ctx.dev_pciids_parse(big.data_ptr(), len(text), stride, nf)
acc = {}
for _ in range(8):
    ctx.set_kernel_timing(True)
    ctx.dev_pciids_parse(big.data_ptr(), len(text), stride, nf)
    for k, v in ctx.kernel_times(): acc.setdefault(k, []).append(v)
ctx.set_kernel_timing(False)
ms = {k: sum(v) / len(v) for k, v in acc.items()}
gb = nf * len(text) / 1e9
print("256 images:", {k: round(v * 1e3, 1) for k, v in ms.items()},
      "scan GB/s %.0f (%.1f%%)  scan+resolve GB/s %.0f" % (gb / (ms["pciids_parse"] * 1e-3), 100 * gb / (ms["pciids_parse"] * 1e-3) / B.peaks()[0],
                                                          gb / ((ms["pciids_parse"] + ms["pciids_resolve"]) * 1e-3)))
# single image
acc = {}
for _ in range(8):
    ctx.set_kernel_timing(True)
    ctx.dev_pciids_parse(d.data_ptr(), len(text), stride, 1)
    for k, v in ctx.kernel_times(): acc.setdefault(k, []).append(v)
ctx.set_kernel_timing(False)
print("   single image us:", {k: round(1e3 * sum(v) / len(v), 1) for k, v in acc.items()})
del big, d
torch.cuda.synchronize(); ctx.close()
