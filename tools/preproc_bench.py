"""Throughput of the GPU image transform (gitb200_preproc_run): Resize(224, bicubic) + CenterCrop(224) + normalise of
64 decoded 480x640 RGB images per call, device-resident source, CUDA events.  HBM-bound byte work: algorithmic bytes per
call = source rows the crop needs (uint8) + fp32 output planes; the uint8 intermediate stays in L2.

    python tools/preproc_bench.py > out/preproc_bench.json
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__  # noqa: E402


def main():
    __graft_entry__.build()
    from generativeimage2text_b200 import _lib, inference as inf
    lib = _lib.load()
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(0)
    t = inf.get_image_transform({})
    t._ensure()
    out_rows = []
    for (h, w, n) in [(480, 640, 64), (1080, 1920, 16), (256, 256, 256)]:
        g = np.random.Generator(np.random.PCG64(1))
        src = torch.from_numpy(g.integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)).to(dev)
        rh, rw, top, left, oh, ow = t.geometry(h, w)
        descs = (_lib.ImageDesc * n)()
        for i in range(n):
            descs[i] = _lib.ImageDesc(i * h * w * 3, h, w, rh, rw, top, left, oh, ow, i * 3 * oh * ow)
        dst = torch.empty((n, 3, oh, ow), dtype=torch.float32, device=dev)
        flush = torch.empty(160 * 1024 * 1024, dtype=torch.uint8, device=dev)
        stream = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(stream):
            def run():
                rc = lib.gitb200_preproc_run(t._handle, src.data_ptr(), src.numel(), 0, descs, n, t._mean, t._std, dst.data_ptr(),
                                             dst.numel(), stream.cuda_stream)
                assert rc == 0, lib.gitb200_preproc_last_error(t._handle)
            for _ in range(3):
                run()
            durs = []
            for _ in range(10):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run()
                e1.record(stream)
                e1.synchronize()
                durs.append(e0.elapsed_time(e1))
        ms = sorted(durs)[len(durs) // 2]
        # rows of the source the vertical windows touch: all of them for a centre crop along the long axis
        src_bytes = n * h * w * 3 if (top == 0) else n * int(h * oh / rh + 12) * w * 3
        alg = src_bytes + dst.numel() * 4
        out_rows.append({'images': n, 'src': [h, w], 'out': [oh, ow], 'ms_per_call': ms, 'images_per_s': n / ms * 1e3,
                         'algorithmic_bytes': alg, 'achieved_gbs': alg / ms / 1e6,
                         'note': 'includes the host-side table build + one H2D of descriptors/weights per call'})
    print(json.dumps(out_rows, indent=1))


if __name__ == '__main__':
    main()
