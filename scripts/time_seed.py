"""Scratch: time the seeding kernel on synthetic 150 bp reads (device-resident).

  python scripts/time_seed.py [n_reads]            syl_seed_batch on ASCII bases (call time)
  python scripts/time_seed.py [n_reads] --packed   syl_sketch_reads_packed2 on 2-bit words: call time and the
                                                    seeding kernel's own time (CUDA events inside the library)
"""
import sys, time
import numpy as np
import torch
sys.path.insert(0, ".")
import sylph_b200
from sylph_b200 import synth
from sylph_b200.api import pack2

args = [a for a in sys.argv[1:] if not a.startswith("--")]
packed = "--packed" in sys.argv
n_reads = int(args[0]) if args else 2_000_000
ctx = sylph_b200.Context(0, stream=torch.cuda.current_stream().cuda_stream)
print("device %s" % torch.cuda.get_device_name(0))
t = time.time()
buf, off = synth.reads(n_reads, device="cuda")
torch.cuda.synchronize()
print("gen %.2fs, %d bases" % (time.time() - t, buf.numel()))
if packed:
    words = torch.from_numpy(pack2(buf.cpu().numpy()).view(np.int32)).cuda()
    n_bases = buf.numel()
    del buf
    ctx.enable_timing(True)
    for it in range(8):
        ctx.seed_kernel_time(reset=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s = ctx.sketch_sequences(words, off, packed_bases=n_bases)
        e1.record(); torch.cuda.synchronize()
        seed_ms, launches, _ = ctx.seed_kernel_time(reset=True)
        print("iter %d: %d k-mers  call %.3f ms  seeding kernel %.3f ms (%d launches)  %.1f Gbase/s"
              % (it, len(s), e0.elapsed_time(e1), seed_ms, launches, n_bases / seed_ms / 1e6))
        s.free()
    ctx.enable_timing(False)
else:
    out = torch.empty(int(buf.numel() / 200 * 1.3 + 4096) * 2, dtype=torch.int64, device="cuda")
    for it in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n = ctx.extract_markers_batch(buf, off, out=out)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        print("iter %d: %d survivors  %.3f ms  %.1f Gbase/s" % (it, n, ms, buf.numel() / ms / 1e6))
