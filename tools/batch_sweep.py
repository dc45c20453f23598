"""Whole-network throughput of the SSCD ResNet-50 (fast mode) as a function of the batch size: tile / wave quantisation of the
persistent kernels (one CTA per SM) makes some batch sizes better operating points than others."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcr_b200 import nets, synthetic   # noqa: E402
from oracle import models as om        # noqa: E402

torch.cuda.set_device(0)
sd = om.make_sscd_state_dict(0)
base = synthetic.images(32, seed=4).cuda()
for batch in [int(a) for a in sys.argv[1:]] or [128, 192, 222, 256, 296, 320, 370, 384, 444, 512]:
    net = nets.build_sscd_resnet50(sd, max_batch=batch, precision="fast")
    img = base.repeat((batch + 31) // 32, 1, 1, 1)[:batch].contiguous()
    for _ in range(3):
        net(img)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(8):
        net(img)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 8
    print(f"batch {batch}: {ms:.3f} ms  {batch / ms * 1e3:.0f} img/s", flush=True)
    del net
    torch.cuda.empty_cache()
