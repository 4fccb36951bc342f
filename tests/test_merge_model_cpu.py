"""The semantics of merge(), pinned on the CPU: a Python model of merge.cpp (candidate order, registries, term order, routes, the newest
holder of a docID deciding, orphan headers, the GOOGLE countdown carried across re-encoded terms only, field statistics) fed through
the host IndexBuilder gives, file for file, the directory the reference's MergeCandidatesCollection::merge() writes over the same
generations.  LUCENE: except the PFor padding the reference leaves uninitialised."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import read_dir
from mergeutil import model_merge, random_specs, ref_merge, write_generation

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
SHAPES = {"one": [G], "one_lucene": [L], "two": [G, G], "three": [G, L, G], "eight": [L, G, L, L, G, G, L, G], "lucene3": [L, L, L]}


def same_but_padding(mine, theirs, what):
    assert mine.size == theirs.size, what
    diff = np.flatnonzero(mine != theirs)
    assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"


def compare_dirs(got_dir, want_dir, codec):
    want, got = read_dir(want_dir), read_dir(got_dir)
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == L and f in ("index", "hits.data"):
            same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f


def build(root, codecs, seed, **kw):
    specs, updated = random_specs(np.random.default_rng(seed), codecs, **kw)
    paths = [root / f"{g + 1}" for g in range(len(codecs))]
    sources = [write_generation(p, c, s, u) for p, c, s, u in zip(paths, codecs, specs, updated)]
    return paths, sources, specs


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
@pytest.mark.parametrize("disable", [False, True], ids=["opt", "noopt"])
@pytest.mark.parametrize("kind", ["plain", "payloads", "freq0"])
def test_model_equals_the_reference(tmp_path, shape, out_codec, disable, kind):
    paths, sources, specs = build(tmp_path / "src", SHAPES[shape], seed=len(shape) * 31 + out_codec, payloads=kind == "payloads", freq0=kind == "freq0")
    index, hits, terms, names, fs = model_merge(out_codec, sources, specs, disable)
    want_fs, _ = ref_merge(out_codec, tmp_path / "ref" / "100", paths, disable, fs["docsCnt"])
    assert fs == want_fs
    tb.segment_write(tmp_path / "model" / "100", out_codec, index, hits if out_codec == L else None, terms, names, fs)
    compare_dirs(tmp_path / "model" / "100", tmp_path / "ref" / "100", out_codec)
