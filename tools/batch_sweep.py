"""How does throughput move with the number of images per engine launch and the number of launches in flight?

The decode loop is a chain of ~45 latency-bound kernels per step whose duration hardly depends on the row count, and
the chains of several batches in flight serialise on the SMs (tools/overlap_sweep.py).  Coalescing k batches of 64 into
ONE decode chain of 64*k rows amortises every kernel boundary and every weight read over k times the rows.  This sweep
measures the BASELINE workload (GIT_BASE, greedy, max_len 40, device-resident pixels) at B images per launch and
`depth` launches in flight:

    GITB200_SLOTS=4 python tools/batch_sweep.py > out/batch_sweep.txt
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault('GITB200_SLOTS', '4')

import torch  # noqa: E402

import __graft_entry__  # noqa: E402


class Tok:
    cls_token_id, sep_token_id = 101, 102


def main():
    __graft_entry__.build()
    from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(0)
    model = get_git_model(Tok(), {})
    model.load_state_dict(synthetic_state_dict({}, 0, 'init'), strict=True)
    model = model.to(dev).eval()
    model.decoder = AutoRegressiveBeamSearch(102, max_steps=40, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    stream = torch.cuda.Stream(device=dev)
    imgs = {B: synthetic_images(B, 0, 1234).contiguous().to(dev) for B in (64, 128, 192, 256)}

    def run(k, depth, img):
        pend, out = [], None
        for _ in range(k):
            if depth == 1:
                out = model({'image': img})
                continue
            pend.append(model.submit({'image': img}, depth=depth))
            if len(pend) >= depth:
                out = pend.pop(0).result()
        while pend:
            out = pend.pop(0).result()
        return out

    rows = []
    for B, depth in [(64, 1), (64, 4), (128, 1), (128, 2), (128, 3), (192, 2), (256, 1), (256, 2), (256, 3)]:
        img = imgs[B]
        n = max(4, 1024 // B)
        with torch.cuda.stream(stream):
            out = run(max(3, 2 * depth), depth, img)
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            out = run(n, depth, img)
            for sl in model._slots:
                if sl['stream'] is not None:
                    stream.wait_stream(sl['stream'])
            e1.record(stream)
            torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1) / n
        assert out['predictions'].shape == (B, 40)
        row = dict(images_per_launch=B, launches_in_flight=depth, ms_per_launch=round(ms, 3),
                   ms_per_64=round(ms * 64 / B, 3), captions_per_s=round(B / ms * 1e3, 1))
        rows.append(row)
        print(json.dumps(row), flush=True)
    print('BEST', json.dumps(max(rows, key=lambda r: r['captions_per_s'])))


if __name__ == '__main__':
    main()
