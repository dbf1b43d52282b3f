"""CPU tests of the sampling contract (tests/sample_ref.py) and of generate's sampling keywords.

  * Philox4x32-10 gives the Random123 known-answer vectors.
  * The reference procedure is a correct sampler: over 2^17 positions of rows of 64 tokens, for a grid of temperature / top-k / top-p,
    its token frequencies pass a chi-square test (p > 1e-6) against the fp64 filtered softmax, and no token outside the kept set is
    ever drawn.
  * Its kept set is the non--inf set of HF's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper (HF's warper order), on
    rows without a near-tie at the top-p boundary, and its probabilities are HF's softmax to 1e-6.
  * Every rejection of the runtime's sampling keywords, raised before anything runs."""
import math

import numpy as np
import pytest

import sample_ref as ref

KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    got = ref.philox(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert tuple(int(v) for v in got) == want


def test_words_layout():
    """Token i at position pos reads word i mod 4 of the block of counter (i / 4, pos, 0, 0) under key (seed lo, seed hi)."""
    seed, pos = 0x0123456789abcdef, 77
    w = ref.words(10, pos, seed)
    for i in range(10):
        blk = ref.philox(np.array([i // 4, pos, 0, 0], dtype=np.uint32), np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32))
        assert w[i] == blk[i % 4]
    u = ref.uniform(np.array([0, 0xFFFFFFFF], dtype=np.uint32))
    assert u[0] == 2.0 ** -24 and u[1] == 1 - 2.0 ** -24 and np.float32(u[1]) == u[1]


GRID = [(1.0, 0, 1.0), (0.7, 0, 1.0), (5.0, 0, 1.0), (1.0, 5, 1.0), (0.7, 0, 0.9), (1.0, 50, 0.5), (0.3, 10, 0.8), (1.0, 1, 1.0),
        (2.0, 0, 1e-6)]


@pytest.mark.parametrize("t,k,p", GRID)
def test_reference_is_a_correct_sampler(t, k, p):
    from scipy import stats
    V, P = 64, 2 ** 17
    x = np.random.default_rng(5).normal(size=V).astype(np.float32) * 2
    x[7] = x[9]  # a tie
    z, _, M = ref.row(x, t, k, p)
    keep = ref.kept(M, z, p)
    want = ref.probs(x, t, k, p)
    s = np.where(keep, z.astype(np.float64) + ref.gumbel(V, np.arange(P), seed=1234), -np.inf)
    tok = np.argmax(s, axis=1)
    counts = np.bincount(tok, minlength=V)
    assert counts[~keep].sum() == 0, "a token outside the kept set was drawn"
    idx = np.flatnonzero(keep)
    if idx.size == 1:
        assert counts[idx[0]] == P
        return
    e = want[idx] * P
    big = e >= 5  # pool the cells of small expected count
    obs = np.append(counts[idx][big], counts[idx][~big].sum())
    exp = np.append(e[big], e[~big].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    assert stats.chisquare(obs, exp).pvalue > 1e-6


def _hf(x, t, k, p):
    torch = pytest.importorskip("torch")
    lp = pytest.importorskip("transformers.generation.logits_process")
    s = torch.from_numpy(x.astype(np.float32))[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    s = lp.TemperatureLogitsWarper(t)(ids, s)
    if k > 0:
        s = lp.TopKLogitsWarper(k)(ids, s)
    if p < 1:
        s = lp.TopPLogitsWarper(p)(ids, s)
    return s[0].double().numpy()


@pytest.mark.parametrize("V", [5, 64, 1000])
@pytest.mark.parametrize("t,k,p", [(1.0, 0, 0.9), (0.7, 20, 1.0), (0.7, 20, 0.8), (1.5, 3, 0.5), (0.5, 0, 0.999), (1.0, 0, 0.3)])
def test_kept_set_is_hf_warpers(V, t, k, p):
    rng = np.random.default_rng(V)
    done = 0
    for _ in range(200):
        x = rng.normal(size=V).astype(np.float32) * 3
        z, _, M = ref.row(x, t, k, p)
        fin = M[np.isfinite(M)]
        if len(np.unique(z)) < V or (p < 1 and np.abs(fin - p).min() < 1e-6):
            continue  # ties or a near-tie at the top-p boundary: HF's sort order and fp32 cumsum decide those
        hf = _hf(x, t, k, p)
        keep = ref.kept(M, z, p)
        assert np.array_equal(keep, np.isfinite(hf))
        hp = np.exp(hf - hf[keep].max())
        hp /= hp.sum()
        assert np.abs(hp - ref.probs(x, t, k, p)).max() < 1e-6
        done += 1
        if done == 10:
            break
    assert done == 10


def test_greedy_rule():
    x = np.array([1, 3, 3, -np.inf], dtype=np.float32)
    assert ref.greedy(x, 0) and ref.greedy(x, -1) and ref.greedy(x, np.nan) and not ref.greedy(x, 0.5)
    assert ref.draw(x, 0, 0, 1, 0, 0) == 1
    assert ref.greedy(np.array([1, np.nan], dtype=np.float32), 1) and ref.greedy(np.array([1, np.inf], dtype=np.float32), 1)
    assert ref.greedy(np.full(4, -np.inf, dtype=np.float32), 1) and ref.greedy(np.array([3e38, 0], dtype=np.float32), 1e-3)


# ---- generate's keywords ------------------------------------------------------------------------------------------------------------
BAD = [
    (dict(temperature=-0.1), "temperature must be a finite number >= 0"),
    (dict(temperature=math.inf), "temperature must be a finite number >= 0"),
    (dict(temperature=math.nan), "temperature must be a finite number >= 0"),
    (dict(temperature="1"), "temperature must be a finite number >= 0"),
    (dict(temperature=True), "temperature must be a finite number >= 0"),
    (dict(temperature=1.0, top_k=-1), "top_k must be an int >= 0"),
    (dict(temperature=1.0, top_k=2.0), "top_k must be an int >= 0"),
    (dict(temperature=1.0, top_k=None), "top_k must be an int >= 0"),
    (dict(temperature=1.0, top_p=0.0), "top_p must be a number in (0, 1]"),
    (dict(temperature=1.0, top_p=1.5), "top_p must be a number in (0, 1]"),
    (dict(temperature=1.0, top_p=-0.5), "top_p must be a number in (0, 1]"),
    (dict(temperature=1.0, top_p=math.nan), "top_p must be a number in (0, 1]"),
    (dict(temperature=1.0, seed=-1), "seed must be an int in [0, 2^63)"),
    (dict(temperature=1.0, seed=2 ** 63), "seed must be an int in [0, 2^63)"),
    (dict(temperature=1.0, seed=1.0), "seed must be an int in [0, 2^63)"),
    (dict(temperature=[1.0, 1.0, 1.0]), "temperature has 3 values for 2 prompt(s)"),
    (dict(temperature=1.0, top_k=[1]), "top_k has 1 values for 2 prompt(s)"),
    (dict(temperature=1.0, top_p=[0.5, 0.5, 0.5]), "top_p has 3 values for 2 prompt(s)"),
    (dict(temperature=1.0, seed=[1, 2, 3]), "seed has 3 values for 2 prompt(s)"),
    (dict(temperature=[1.0, -1.0]), "temperature must be a finite number >= 0"),
    (dict(temperature=1.0, seed=2 ** 63 - 1), "seed must be an int in [0, 2^63) (got 9223372036854775808)"),  # s + 1 for prompt 1
]


@pytest.mark.parametrize("kw,frag", BAD, ids=[f"{i}" for i in range(len(BAD))])
def test_sampling_keywords_rejected(kw, frag):
    from squeezellm_b200.runtime import _sampling
    with pytest.raises(ValueError, match=re_escape(frag)):
        _sampling("X.generate", 2, **{**dict(temperature=0.0, top_k=0, top_p=1.0, seed=0), **kw})


def re_escape(s):
    import re
    return re.escape(s)


def test_sampling_keywords_accepted():
    from squeezellm_b200.runtime import _sampling
    assert _sampling("X", 3, 0.0, 5, 0.5, 7) is None  # every temperature 0: greedy, no sampler
    assert _sampling("X", 2, [0, 0.0], 0, 1.0, 0) is None
    t, k, p, s = _sampling("X", 3, 0.7, 2 ** 40, 0.9, 5)
    assert t == [0.7] * 3 and k == [2 ** 31 - 1] * 3 and p == [0.9] * 3 and s == [5, 6, 7]
    t, k, p, s = _sampling("X", 2, [0.0, 1.0], [0, 3], [1.0, 0.5], [9, 9])
    assert t == [0.0, 1.0] and k == [0, 3] and p == [1.0, 0.5] and s == [9, 9]
    assert _sampling("X", 1, np.float32(0.5), np.int64(4), 1, np.int64(3)) is not None


def test_generate_rejects_before_anything_runs():
    """The keywords are checked first: on a decoder object with no state at all the ValueError comes before any attribute is read."""
    from squeezellm_b200.runtime import BatchDecoder, SequenceDecoder
    with pytest.raises(ValueError, match="SequenceDecoder.generate: top_p must be"):
        object.__new__(SequenceDecoder).generate([1, 2], 4, temperature=1.0, top_p=2.0)
    dec = object.__new__(BatchDecoder)
    dec.batch = 4
    with pytest.raises(ValueError, match=re_escape("BatchDecoder.generate: seed has 1 values for 2 prompt(s)")):
        dec.generate([[1, 2], [3]], 4, temperature=1.0, seed=[1])
