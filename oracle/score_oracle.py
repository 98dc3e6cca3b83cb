"""TEST INFRASTRUCTURE ONLY -- CPU restatement (fp32, plain torch ops) of the reference's caption-scoring forward: the
training branch of CaptioningModel.forward_one_ce (layers/decoder.py:916-972) with dropout off, which
GitB200CaptioningModel.score implements on the GPU.  Built from the pieces of git_oracle.py; pinned against the unmodified
reference by tests/golden/score_*.npz (oracle/make_score_golden.py, tests/test_score_host.py).  The product package never
imports it.
"""
import torch
import torch.nn.functional as F

from git_oracle import DEC_LAYERS, _bert_layer, _kv, embed_tokens, lm_head, project_visual, visual_features


def smooth_label_ce(logits, target, eps=0.1):
    """SmoothLabelCrossEntropyLoss (layers/decoder.py:620-671) on rows that are already filtered: KL(one_hot_eps || softmax)
    summed over classes, mean over rows."""
    n_class = logits.shape[1]
    one_hot = torch.zeros_like(logits).scatter(1, target.view(-1, 1), 1)
    one_hot = one_hot * (1 - eps) + (1 - one_hot) * eps / (n_class - 1)
    lp = F.log_softmax(logits, dim=1)
    return (one_hot * (one_hot.log() - lp)).sum(dim=1).mean()


@torch.no_grad()
def score_captions(sd, param, batch, cols=None):
    """CaptioningModel.forward_one_ce, training branch (layers/decoder.py:916-972), without dropout: the visual features of
    each image, visual_projection, embed_tokens over the T positions, 6 x _bert_layer over [image || text] with the block
    mask of as_shipped_step (layers/decoder.py:114-137, 602-610), lm_head on every text row, then log-softmax / gather and
    SmoothLabelCrossEntropyLoss over the positions with need_predict[:, t+1] == 1 and a non-zero target (:937-960).

    batch: {'image': tensor [B,3,H,W] | list of frames | list of [3,H_b,W_b] images, 'caption_tokens' [N,T],
            'need_predict' [N,T], 'image_index'? [N]}.  Caption n uses image image_index[n] (default n).
    Returns {'token_logprobs' [N, T-1], 'vl_l_loss' scalar, 'logits' [N, T, len(cols)] when cols is given}."""
    image = batch['image']
    tokens = torch.as_tensor(batch['caption_tokens']).long()
    need = torch.as_tensor(batch['need_predict']).long()
    N, T = tokens.shape
    ragged = isinstance(image, (list, tuple)) and image[0].dim() == 3
    if ragged:
        feats = [visual_features(sd, param, im[None]) for im in image]
    else:
        f = visual_features(sd, param, image)
        feats = [f[b:b + 1] for b in range(f.shape[0])]
    index = batch.get('image_index')
    index = list(range(N)) if index is None else [int(i) for i in index]
    logits = torch.zeros(N, T, 30522) if cols is None else None
    lp_all = torch.zeros(N, T - 1)
    col_logits = torch.zeros(N, T, len(cols)) if cols is not None else None
    feat_rows = []
    for b in sorted(set(index)):
        rows = [n for n in range(N) if index[n] == b]
        v = project_visual(sd, feats[b]).expand(len(rows), -1, -1)
        e = embed_tokens(sd, tokens[rows])
        M = v.shape[1]
        x = torch.cat([v, e], dim=1)
        mask = torch.zeros(M + T, M + T)
        mask[:M, M:] = float('-inf')
        mask[M:, M:] = torch.triu(torch.full((T, T), float('-inf')), diagonal=1)
        mask = mask[None, None]
        for j in range(DEC_LAYERS):
            k, vv = _kv(sd, j, x)
            x = _bert_layer(sd, j, x, k, vv, mask)
        z = lm_head(sd, x[:, M:])                                                 # [rows, T, V]
        lp = F.log_softmax(z[:, :-1], dim=-1).gather(2, tokens[rows, 1:, None])[..., 0]
        lp_all[rows] = lp
        if cols is not None:
            col_logits[rows] = z[:, :, torch.as_tensor(cols)]
        else:
            logits[rows] = z
        feat_rows.append((rows, z))
    valid = (need[:, 1:] == 1) & (tokens[:, 1:] != 0)
    feat, target = [], []
    for rows, z in feat_rows:
        vm = valid[rows]
        feat.append(z[:, :-1][vm])
        target.append(tokens[rows, 1:][vm])
    loss = smooth_label_ce(torch.cat(feat), torch.cat(target))
    out = {'token_logprobs': lp_all, 'vl_l_loss': loss}
    out['logits'] = col_logits if cols is not None else logits
    return out
