"""The decode loop's captured step graphs and the one-call inputs of the C API, checked against a fresh engine.

A step graph bakes in buffer addresses and the call's search context, so an engine may replay one only for a call whose
launches would be the same: after calls of other sizes (the serving path coalesces batches into launches of different
row counts) and after gitb200_set_trie re-allocates the trie's edge buffers.  The inputs set for the next call
(gitb200_set_row_prefixes, gitb200_set_sampling) are taken by that call even when it fails.  Every result here must be
bit-identical to what a newly created engine returns for the same inputs."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_STEPS = 10
EOS = 102


class Tok:
    cls_token_id, sep_token_id = 101, 102


@pytest.fixture(scope='module')
def state_dict():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    return synthetic_state_dict({}, 0, 'perturbed')


def _model(sd, search='greedy', trie=None):
    from generativeimage2text_b200.model import (get_git_model, AutoRegressiveBeamSearch, GeneratorWithBeamSearch,
                                                 TrieAutoRegressiveBeamSearch)
    m = get_git_model(Tok(), {})
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    if trie is not None:
        m.decoder = TrieAutoRegressiveBeamSearch(EOS, max_steps=MAX_STEPS, beam_size=1, trie=trie)
    elif search == 'greedy':
        m.decoder = AutoRegressiveBeamSearch(EOS, max_steps=MAX_STEPS, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    else:
        m.decoder = GeneratorWithBeamSearch(EOS, max_steps=MAX_STEPS, beam_size=4, length_penalty=0.6)
    return m


def _images(n, seed):
    from generativeimage2text_b200.synthetic import synthetic_images
    return synthetic_images(n, 0, seed).cuda()


def _assert_same(got, want):
    torch.cuda.synchronize()
    assert torch.equal(got['predictions'], want['predictions'])
    assert torch.equal(got['logprobs'].reshape(-1), want['logprobs'].reshape(-1))


@pytest.mark.parametrize('search,sizes', [('greedy', (64, 128, 64)), ('beam', (32, 64, 32))])
def test_calls_of_other_sizes_on_one_engine_match_a_fresh_engine(state_dict, search, sizes):
    """Calls that grow the engine's buffers and then shrink back (greedy: the one-kernel step at 64 rows, the kernel chain
    at 128; beam: 4 beams per image) give what a fresh engine gives for each call."""
    m, fresh = _model(state_dict, search), _model(state_dict, search)
    for i, n in enumerate(sizes):
        img = _images(n, 300 + i)
        got = m({'image': img})
        fresh.release()                 # a new engine for every call
        _assert_same(got, fresh({'image': img}))


class _Csr(object):
    """A trie in the CSR form gitb200_set_trie takes, for the model's trie decoder."""

    def __init__(self, begin, token, child):
        self.csr = (begin, token, child)

    def to_csr(self):
        return self.csr


def _more_edges(begin, token, child, vocab=30522):
    """The same nodes with one more edge out of every node: to the root, by a token the node did not accept."""
    nb, nt, nc = [0], [], []
    for v in range(len(begin) - 1):
        own = token[begin[v]:begin[v + 1]]
        nt += own
        nc += child[begin[v]:begin[v + 1]]
        nt.append(next(t for t in range(1000, vocab) if t not in own))
        nc.append(0)
        nb.append(len(nt))
    return _Csr(nb, nt, nc)


def test_a_trie_with_more_edges_after_a_constrained_call_matches_a_fresh_engine(state_dict):
    """gitb200_set_trie with the node count of the trie the last call ran under and more edges re-allocates the edge
    buffers that call's step graph read; the next call must run under the new trie."""
    from generativeimage2text_b200.model import TokenTrie, TrieAutoRegressiveBeamSearch
    img = _images(8, 77)
    m = _model(state_dict)
    free = m({'image': img})['predictions'].cpu()
    trie = TokenTrie.construct([[t for t in row[1:] if t != EOS][:3] + [EOS] for row in free.tolist()])
    m.decoder = TrieAutoRegressiveBeamSearch(EOS, max_steps=MAX_STEPS, beam_size=1, trie=trie)
    m({'image': img})
    wider = _more_edges(*trie.to_csr())
    assert len(wider.csr[0]) == len(trie.to_csr()[0]) and len(wider.csr[1]) > len(trie.to_csr()[1])
    m.decoder = TrieAutoRegressiveBeamSearch(EOS, max_steps=MAX_STEPS, beam_size=1, trie=wider)   # set through the C API
    got = m({'image': img})
    _assert_same(got, _model(state_dict, trie=wider)({'image': img}))


@pytest.mark.parametrize('pending', ['row_prefixes', 'sampling'])
def test_a_call_that_fails_validation_leaves_no_one_call_input_behind(state_dict, pending):
    """An input set for the next call is taken by that call even when it then fails: the call after it runs without it."""
    from generativeimage2text_b200 import _lib
    lib = _lib.load()
    img = _images(4, 91)
    B = img.shape[0]
    m = _model(state_dict)
    m({'image': img})
    eng = m._engine
    prefix = torch.tensor([[101, 2054, 2003]] * B, dtype=torch.long, device='cuda')
    lens = torch.full((B,), 2, dtype=torch.int32, device='cuda')
    uniforms = torch.rand((MAX_STEPS, B), generator=torch.Generator().manual_seed(5)).cuda()
    if pending == 'row_prefixes':
        _lib.check(lib.gitb200_set_row_prefixes(eng, prefix.data_ptr(), B, prefix.shape[1], lens.data_ptr()), eng, 'set_row_prefixes')
    else:
        _lib.check(lib.gitb200_set_sampling(eng, uniforms.data_ptr(), MAX_STEPS, B, 0.7), eng, 'set_sampling')
    sp = m._search_struct()
    logprobs = torch.empty((B,), dtype=torch.float32, device='cuda')
    rc = lib.gitb200_generate(eng, img.data_ptr(), B, 0, None, 0, ctypes.byref(sp), None, None, logprobs.data_ptr(),
                              None, None, None)
    assert rc != 0 and b'null buffer' in lib.gitb200_last_error(eng)
    got = m({'image': img})
    _assert_same(got, _model(state_dict)({'image': img}))
