"""CPU: host logic of generativeimage2text_b200/model.py that needs no device -- the per-batch views a coalesced engine
launch hands back (`_Group` / `_Member`, `greedy_width`), against what the reference's loops would have returned for each
batch alone (reference layers/decoder.py:279-291, 316-320, 433-438)."""
import warnings

import pytest
import torch

from generativeimage2text_b200 import model as M

EOS = 102


def test_greedy_width_is_where_the_reference_loop_stops():
    # the reference appends a column, then stops before the next step once EVERY row's last token is EOS
    p = torch.tensor([[101, 5, 6, EOS, EOS, EOS], [101, 7, EOS, EOS, EOS, EOS]])
    assert M.greedy_width(p, EOS) == 4
    assert M.greedy_width(torch.tensor([[101, 5, 6, 7], [101, 7, EOS, EOS]]), EOS) == 4      # never all-EOS: full width
    assert M.greedy_width(torch.tensor([[101, 5, EOS], [101, 9, EOS]]), EOS) == 3


class _FakePending:
    def __init__(self, out):
        self.out = out

    def result(self):
        return self.out


class _FakeModel:
    """Stands in for GitB200CaptioningModel: records what a group launches and returns a canned engine result."""

    def __init__(self, decoder, out):
        self.decoder, self.eos_index, self._open_group, self.out = decoder, EOS, None, out
        self.launched = []

    def submit(self, batch, depth=2):
        self.launched.append(batch['image'])
        return _FakePending(self.out)


def _rec(x, frames=0):
    """The images of one batch as GitB200CaptioningModel._image_batch records them (x: [B, 3, H, W] or [frames, B, 3, H, W])."""
    B = int(x.shape[-4])
    return M._Images(x, B, frames, None, [1] * B)


def _greedy():
    return M.AutoRegressiveBeamSearch(EOS, max_steps=6, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)


def test_members_of_coalesced_image_records_get_their_own_rows_widths_and_the_empty_caption_exit():
    toks = torch.tensor([
        [101, 11, 12, 13, 14, 15],      # batch 0 (2 rows): never finishes -> full width
        [101, 21, EOS, EOS, EOS, EOS],
        [101, 31, 32, EOS, EOS, EOS],   # batch 1 (2 rows): all EOS from column 3 -> width 4
        [101, 41, EOS, EOS, EOS, EOS],
        [101, EOS, EOS, EOS, EOS, EOS],  # batch 2 (1 row): first token EOS -> the reference's empty-caption exit
    ])
    lps = torch.tensor([-1.0, -2.0, -3.0, -4.0, -5.0])
    fm = _FakeModel(_greedy(), {'predictions': toks, 'logprobs': lps})
    g = M._Group(fm, key=('k',), depth=2, want=3)
    fm._open_group = g
    imgs = [torch.zeros(2, 3, 4, 4), torch.ones(2, 3, 4, 4), torch.full((1, 3, 4, 4), 2.0)]
    members = [M._Member(g, g.add(_rec(im))) for im in imgs]
    g.launch()
    assert fm._open_group is None and len(fm.launched) == 1
    cat = fm.launched[0]
    assert cat.B == 5 and cat.frames == 0
    assert cat.x.shape == (5, 3, 4, 4) and float(cat.x[2:4].mean()) == 1.0                       # concatenated in order
    g.launch()                                                                                   # idempotent
    assert len(fm.launched) == 1
    a = members[0].result()
    assert a['predictions'].tolist() == toks[0:2].tolist() and a['logprobs'].tolist() == [-1.0, -2.0]
    b = members[1].result()
    assert b['predictions'].tolist() == toks[2:4, :4].tolist() and b['logprobs'].tolist() == [-3.0, -4.0]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        c = members[2].result()
    assert any('Empty captions' in str(x.message) for x in w)
    assert c['predictions'].tolist() == [[EOS]] and tuple(c['logprobs'].shape) == (1, 1) and float(c['logprobs']) == -5.0
    assert members[1].result() is b                                                              # cached


def test_video_records_are_concatenated_along_the_batch_axis_and_beam_results_are_sliced():
    beam = M.GeneratorWithBeamSearch(EOS, max_steps=4, beam_size=4, length_penalty=0.6)
    toks = torch.arange(12).reshape(3, 4)
    lps = torch.tensor([[-0.1], [-0.2], [-0.3]])
    fm = _FakeModel(beam, {'predictions': toks, 'logprobs': lps})
    g = M._Group(fm, key=('k',), depth=2, want=2)
    a = torch.stack([torch.zeros(1, 3, 2, 2), torch.zeros(1, 3, 2, 2) + 1])          # 2 frames, 1 image
    b = torch.stack([torch.zeros(2, 3, 2, 2) + 5, torch.zeros(2, 3, 2, 2) + 6])      # 2 frames, 2 images
    ma, mb = M._Member(g, g.add(_rec(a, 2))), M._Member(g, g.add(_rec(b, 2)))
    ra = ma.result()                                                   # asking for a result launches the group
    cat = fm.launched[0]
    assert cat.frames == 2 and cat.B == 3 and cat.x.shape == (2, 3, 3, 2, 2)
    assert cat.x[0][:, 0, 0, 0].tolist() == [0.0, 5.0, 5.0] and cat.x[1][:, 0, 0, 0].tolist() == [1.0, 6.0, 6.0]
    assert ra['predictions'].tolist() == toks[0:1].tolist() and tuple(ra['logprobs'].shape) == (1, 1)
    assert mb.result()['predictions'].tolist() == toks[1:3].tolist()


def test_search_configuration_classes_keep_the_reference_checks():
    with pytest.raises(AssertionError):
        M.AutoRegressiveBeamSearch(EOS, max_steps=8, beam_size=1, per_node_beam_size=1, fix_missing_prefix=False)
    with pytest.raises(NotImplementedError):
        M.AutoRegressiveBeamSearch(EOS, max_steps=8, beam_size=5, per_node_beam_size=2, fix_missing_prefix=True)
    with pytest.raises(AssertionError):
        M.GeneratorWithBeamSearch(EOS, max_steps=8, beam_size=4, length_penalty=0)
    with pytest.raises(NotImplementedError):
        M.GeneratorWithBeamSearch(EOS, max_steps=8, beam_size=4, temperature=0.7)


def test_token_trie_mirror_and_csr():
    """TokenTrie (reference trie_decoder.py:224-258) mirror: same answers as a plain prefix scan; CSR export round-trips."""
    import random
    from generativeimage2text_b200.model import TokenTrie, TrieAutoRegressiveBeamSearch
    rnd = random.Random(4)
    seqs = [[rnd.randrange(0, 12) for _ in range(rnd.randrange(1, 6))] + [102] for _ in range(60)]
    trie = TokenTrie.construct(seqs)
    for _ in range(200):
        pre = rnd.choice(seqs)[:rnd.randrange(0, 5)]
        want = sorted({s[len(pre)] for s in seqs if s[:len(pre)] == pre and len(s) > len(pre)})
        assert sorted(trie.get_valid(pre)) == want
    begin, tok, child = trie.to_csr()
    assert begin[0] == 0 and begin[-1] == len(tok) == len(child)
    for s in seqs:                                            # every sequence is a root-to-leaf walk of the CSR form
        node = 0
        for t in s:
            edges = range(begin[node], begin[node + 1])
            hit = [e for e in edges if tok[e] == t]
            assert len(hit) == 1
            node = child[hit[0]]
    trie.reset()
    trie.move(seqs[0][0])
    assert sorted(trie.get_curr_valid()) == sorted(trie.get_valid(seqs[0][:1]))
    d = TrieAutoRegressiveBeamSearch(102, max_steps=20, beam_size=1, trie=trie)
    assert d.per_node_beam_size == 1 and d.trie is trie
    import pytest
    with pytest.raises(AssertionError):
        TrieAutoRegressiveBeamSearch(102, max_steps=20, beam_size=2, trie=trie)      # reference trie_decoder.py:38


def test_search_param_validation_mirrors_the_reference_signature():
    """`search_param` is what CaptioningModel.infer forwards to decoder.search (reference layers/decoder.py:999-1003, 224-232):
    the host-side checks of `_sampling_setup`, on the CPU (no engine is touched)."""
    import types
    from generativeimage2text_b200 import _lib

    class Tok:
        cls_token_id, sep_token_id = 101, 102
    m = M.get_git_model(Tok(), {})
    sp = _lib.Search(mode=_lib.SEARCH_GREEDY, max_steps=12, beam_size=1, per_node_beam=1, length_penalty=1.0)
    cpu = torch.device('cpu')
    m.decoder = M.AutoRegressiveBeamSearch(EOS, max_steps=12, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    assert m._sampling_setup({}, sp, 3, cpu) is None
    assert m._sampling_setup({'do_sample': False}, sp, 3, cpu) is None
    u = m._sampling_setup({'do_sample': True, 'temperature': 0.7, 'top_k': 5, 'top_p': 0.9}, sp, 3, cpu)     # top_k / top_p: ignored
    assert tuple(u.shape) == (12, 3) and u.dtype == torch.float32 and bool(((u >= 0) & (u < 1)).all())
    g1 = m._sampling_setup({'do_sample': True, 'generator': torch.Generator().manual_seed(7)}, sp, 3, cpu)
    g2 = m._sampling_setup({'do_sample': True, 'generator': torch.Generator().manual_seed(7)}, sp, 3, cpu)
    assert torch.equal(g1, g2)
    mine = torch.rand(14, 3)
    assert m._sampling_setup({'do_sample': True, 'uniforms': mine}, sp, 3, cpu) is not None
    with pytest.raises(ValueError):
        m._sampling_setup({'do_sample': True, 'uniforms': torch.rand(5, 3)}, sp, 3, cpu)          # fewer than max_steps rows
    with pytest.raises(ValueError):
        m._sampling_setup({'do_sample': True, 'temperature': 0.0}, sp, 3, cpu)
    with pytest.raises(AssertionError):
        m._sampling_setup({'temperature': 0.5}, sp, 3, cpu)                                        # reference :259-261
    with pytest.raises(TypeError):
        m._sampling_setup({'do_sample': True, 'beam_width': 3}, sp, 3, cpu)
    with pytest.raises(NotImplementedError):
        m._sampling_setup({'do_sample': True, 'num_return_sequences': 2}, sp, 3, cpu)
    m.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=12, beam_size=4, length_penalty=0.6)
    with pytest.raises(NotImplementedError):
        m._sampling_setup({'do_sample': True}, sp, 3, cpu)
    # the trie decoder maps onto the greedy search mode of the engine
    m.decoder = M.TrieAutoRegressiveBeamSearch(EOS, max_steps=9, beam_size=1, trie=M.TokenTrie.construct([[5, EOS]]))
    s2 = m._search_struct()
    assert s2.mode == _lib.SEARCH_GREEDY and s2.max_steps == 9 and s2.beam_size == 1
    m.decoder = types.SimpleNamespace()
    with pytest.raises(TypeError):
        m._search_struct()
