"""A/B of the persistent one-kernel decode step against the kernel chain on whole model(batch) calls:
    python tools/mega_ab.py [rows ...] > out/mega_ab.txt"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images


class Tok:
    cls_token_id, sep_token_id = 101, 102


rows_list = [int(a) for a in sys.argv[1:]] or [64, 16]
m = get_git_model(Tok(), {})
m.load_state_dict(synthetic_state_dict({}, 0, 'init'))
m = m.cuda().eval()
m.decoder = AutoRegressiveBeamSearch(102, max_steps=40, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
s = torch.cuda.Stream()
with torch.cuda.stream(s):
    for rows in rows_list:
        img = synthetic_images(rows).cuda()
        ref = None
        for opts in ({'use_mega': 1}, {'use_mega': 0}, {'use_mega': 1}):
            for k, v in opts.items():
                m.set_engine_option(k, v)
            for _ in range(2):
                out = m({'image': img})
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            n = 6
            for _ in range(n):
                out = m({'image': img})
            e1.record(s)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n
            if ref is None:
                ref = out['predictions'].clone()
            agree = float((out['predictions'] == ref).float().mean())
            print(json.dumps(dict(rows=rows, **opts, ms_per_call=round(ms, 3), captions_per_s=round(rows / ms * 1e3, 1),
                                  token_agreement_with_first=round(agree, 4))), flush=True)
