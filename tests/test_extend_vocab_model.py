"""C2V_EXTEND_VOCAB=1 on the host: the merge rule of vocabularies.extend_vocab against a plain statement of it over
pickled dictionaries, the switch and its refusal, and multi_rank's row reader filling taller shards and target blocks
than the checkpoint's tables (DESIGN.md §6m)."""
import os
import pickle

import numpy as np
import pytest

from code2vec_b200.config import Config
from code2vec_b200.vocabularies import Code2VecVocabs, Vocab, VocabType, extend_vocab

SLOTS = ((VocabType.Token, "token_vocab", "MAX_TOKEN_VOCAB_SIZE"), (VocabType.Path, "path_vocab", "MAX_PATH_VOCAB_SIZE"),
         (VocabType.Target, "target_vocab", "MAX_TARGET_VOCAB_SIZE"))


def _statement(loaded_words, specials, counts, cap):
    """The rule in plain Python: index -> word of the loaded vocabulary (specials first), then the words of the
    from-scratch vocabulary (count descending, ties in dict order, at most `cap`) that it lacks, in that order."""
    out = list(specials) + list(loaded_words)
    ranked = sorted(counts, key=lambda w: -counts[w])[:cap]      # sorted() is stable
    for w in list(specials) + ranked:
        if w not in out:
            out.append(w)
    return out


def _write_model(tmp_path, separate, vocab_words):
    """dictionaries.bin of a model whose vocabularies hold `vocab_words` (token, path, target lists), and its folder."""
    cfg = _cfg(tmp_path, separate)
    folder = tmp_path / "old"
    folder.mkdir(exist_ok=True)
    vocabs = Code2VecVocabs.__new__(Code2VecVocabs)
    vocabs.config, vocabs._already_saved_in_paths = cfg, set()
    for (kind, attr, _), words in zip(SLOTS, vocab_words):
        setattr(vocabs, attr, Vocab(kind, words, vocabs._get_special_words_by_vocab_type(kind)))
    vocabs.save(str(folder / "dictionaries.bin"))
    return str(folder / "saved")


def _write_dataset(tmp_path, histograms, name="new"):
    prefix = str(tmp_path / name)
    with open(prefix + ".dict.c2v", "wb") as f:
        for h in histograms:                                       # token, path, target, then the example count
            pickle.dump(h, f)
        pickle.dump(10, f)
    return prefix


def _cfg(tmp_path, separate=False, **kw):
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.SEPARATE_OOV_AND_PAD = separate
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


LOADED = (["a", "b", "c", "d"], ["10", "11", "12"], ["get|x", "set|x"])
NEW = ({"c": 9, "e": 9, "f": 3, "a": 50, "g": 9, "h": 1}, {"13": 2, "11": 5, "14": 2, "15": 1}, {"run": 4, "get|x": 7, "is|y": 4})


@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("caps", [(1000, 1000, 1000), (4, 2, 1)])
def test_merge_rule_against_statement(tmp_path, separate, caps):
    load = _write_model(tmp_path, separate, LOADED)
    prefix = _write_dataset(tmp_path, NEW)
    cfg = _cfg(tmp_path, separate, MODEL_LOAD_PATH=load, TRAIN_DATA_PATH_PREFIX=prefix, MAX_TOKEN_VOCAB_SIZE=caps[0],
               MAX_PATH_VOCAB_SIZE=caps[1], MAX_TARGET_VOCAB_SIZE=caps[2])
    plain = Code2VecVocabs(cfg)
    grown = Code2VecVocabs(cfg, extend=True)
    assert plain.loaded_sizes is None
    for (kind, attr, limit), loaded_words, counts in zip(SLOTS, LOADED, NEW):
        old, new = getattr(plain, attr), getattr(grown, attr)
        specials = list(dict.fromkeys(vars(old.special_words).values()))
        want = _statement(loaded_words, specials, counts, getattr(cfg, limit))
        assert [new.index_to_word[i] for i in range(new.size)] == want, kind
        assert new.word_to_index == {w: i for i, w in enumerate(want)}
        assert grown.loaded_sizes[kind] == old.size
        for w, i in old.word_to_index.items():                    # old indices unchanged
            assert new.word_to_index[w] == i
        assert len(set(want)) == len(want)                        # no special (or other) word twice
    # the cap: (4, 2, 1) keeps a, c, e, g of the tokens (ties c, e, g in dict order) and adds e, g
    if caps == (4, 2, 1):
        assert [grown.token_vocab.index_to_word[i] for i in range(plain.token_vocab.size, grown.token_vocab.size)] == ["e", "g"]
        assert grown.target_vocab.size == plain.target_vocab.size          # its one word, get|x, is already held


def test_all_words_known_gives_loaded_vocabularies(tmp_path):
    load = _write_model(tmp_path, False, LOADED)
    prefix = _write_dataset(tmp_path, ({"b": 3, "a": 1}, {"12": 1}, {"set|x": 2}))
    cfg = _cfg(tmp_path, MODEL_LOAD_PATH=load, TRAIN_DATA_PATH_PREFIX=prefix)
    plain, grown = Code2VecVocabs(cfg), Code2VecVocabs(cfg, extend=True)
    for _, attr, _ in SLOTS:
        a, b = getattr(plain, attr), getattr(grown, attr)
        assert (a.size, a.word_to_index, a.index_to_word) == (b.size, b.word_to_index, b.index_to_word)
    # saved, the merged vocabularies are the loaded file byte for byte
    out = tmp_path / "out"
    out.mkdir()
    grown.save(str(out / "dictionaries.bin"))
    assert open(str(out / "dictionaries.bin"), "rb").read() == open(str(tmp_path / "old" / "dictionaries.bin"), "rb").read()


def test_saved_merged_vocabularies_load_back(tmp_path):
    load = _write_model(tmp_path, True, LOADED)
    prefix = _write_dataset(tmp_path, NEW)
    grown = Code2VecVocabs(_cfg(tmp_path, True, MODEL_LOAD_PATH=load, TRAIN_DATA_PATH_PREFIX=prefix), extend=True)
    out = tmp_path / "out"
    out.mkdir()
    grown.save(str(out / "dictionaries.bin"))
    again = Code2VecVocabs(_cfg(tmp_path, True, MODEL_LOAD_PATH=str(out / "saved")))
    for _, attr, _ in SLOTS:
        a, b = getattr(grown, attr), getattr(again, attr)
        assert (a.size, a.word_to_index, a.index_to_word) == (b.size, b.word_to_index, b.index_to_word)


def test_extend_vocab_is_the_rule_on_one_vocab():
    specials = Code2VecVocabs.__new__(Code2VecVocabs)
    specials.config = _cfg(None, True)
    sw = specials._get_special_words_by_vocab_type(VocabType.Token)
    loaded = Vocab(VocabType.Token, ["x", "y"], sw)
    merged = extend_vocab(loaded, {"<PAD>": 5, "z": 5, "y": 4, "w": 6}, 3)
    assert [merged.index_to_word[i] for i in range(merged.size)] == ["<PAD>", "<OOV>", "x", "y", "w", "z"]
    assert loaded.size == 4 and "w" not in loaded.word_to_index          # the loaded vocabulary is left as it was


# ---- the switch -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("raw, want", [("", False), ("0", False), ("1", True)])
def test_flag_values(raw, want):
    from code2vec_b200.b200_model import extend_vocab_flag
    assert extend_vocab_flag({"C2V_EXTEND_VOCAB": raw}) is want
    assert extend_vocab_flag({}) is False


@pytest.mark.parametrize("raw", ["2", "yes", " 1", "true"])
def test_flag_refuses_other_values(raw):
    from code2vec_b200.b200_model import extend_vocab_flag
    with pytest.raises(ValueError, match=r"C2V_EXTEND_VOCAB must be 0 or 1, got %r" % raw):
        extend_vocab_flag({"C2V_EXTEND_VOCAB": raw})


def test_no_effect_log_lines(tmp_path):
    from code2vec_b200.b200_model import extend_vocab_run
    lines = []
    cfg = _cfg(tmp_path, MODEL_LOAD_PATH=str(tmp_path / "m" / "saved"), TEST_DATA_PATH="t.c2v")
    assert extend_vocab_run(cfg, True, lines.append) is False
    assert lines == ["C2V_EXTEND_VOCAB=1 has no effect: this run does not train (no --data)"]
    lines.clear()
    cfg = _cfg(tmp_path, TRAIN_DATA_PATH_PREFIX="d", MODEL_SAVE_PATH=str(tmp_path / "saved"))
    assert extend_vocab_run(cfg, True, lines.append) is False
    assert lines == ["C2V_EXTEND_VOCAB=1 has no effect: this run does not load a model (no --load), and a model trained "
                     "from scratch already takes the dataset's vocabulary"]
    lines.clear()
    cfg = _cfg(tmp_path, TRAIN_DATA_PATH_PREFIX="d", MODEL_LOAD_PATH=str(tmp_path / "a" / "saved"),
               MODEL_SAVE_PATH=str(tmp_path / "b" / "saved"))
    assert extend_vocab_run(cfg, True, lines.append) is True and lines == []
    assert extend_vocab_run(cfg, False, lines.append) is False and lines == []


@pytest.mark.parametrize("save", ["m/other_name", "m/./saved_iter8", "link/saved"])
def test_same_directory_refused_before_any_file_is_touched(tmp_path, monkeypatch, save):
    """--save into the --load directory (by another name, a dotted path, or a link to it): ValueError naming the
    dictionaries.bin it would replace, raised by Code2VecModel before it writes a side-car, a log file or anything else."""
    from code2vec_b200 import load_model_dynamically
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_EXTEND_VOCAB", "1")
    load = _write_model(tmp_path, False, LOADED)
    os.rename(str(tmp_path / "old"), str(tmp_path / "m"))
    os.symlink(str(tmp_path / "m"), str(tmp_path / "link"))
    prefix = _write_dataset(tmp_path, NEW)
    with open(prefix + ".train.c2v", "w") as f:
        f.write("get|x a,10,b\n")
    before = {p: os.stat(os.path.join(dp, p)).st_mtime_ns for dp, _, fs in os.walk(str(tmp_path)) for p in fs}
    for framework in ("b200", "b200-keras"):
        cfg = _cfg(tmp_path, DL_FRAMEWORK=framework, MODEL_LOAD_PATH="m/saved", TRAIN_DATA_PATH_PREFIX=prefix,
                   MODEL_SAVE_PATH=save, LOGS_PATH=str(tmp_path / "run.log"))
        with pytest.raises(ValueError) as err:
            load_model_dynamically(cfg)
        assert str(err.value).startswith("C2V_EXTEND_VOCAB=1: --save writes the extended vocabularies to `%s`" %
                                         os.path.join(os.path.realpath(str(tmp_path / "m")), "dictionaries.bin")), str(err.value)
    after = {p: os.stat(os.path.join(dp, p)).st_mtime_ns for dp, _, fs in os.walk(str(tmp_path)) for p in fs}
    assert after == before
    del load


# ---- the sharded row reader into taller shards ------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_sharded_reader_fills_taller_shards(tmp_path, world):
    """A checkpoint of T_old = 1001 token rows (and Y_old target rows) read into the shards and target blocks of a model
    grown to T_new = 1100 (Y_new): each rank's rows below the old sizes come from the file, every other row is left as
    it was, including target blocks that straddle Y_old or lie wholly past it."""
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.multi_rank import checkpoint_header, read_checkpoint_part, write_checkpoint
    from code2vec_b200.trainer import target_row_block
    T_old, T_new, P_old, P_new, Y_old, Y_new, d, D = 1001, 1100, 37, 40, 21, 34, 4, 6
    old = EngineDims(token_vocab=T_old, path_vocab=P_old, target_vocab=Y_old, embed_dim=d, code_dim=D, max_contexts=3,
                     max_batch=8)
    rng = np.random.default_rng(world)
    full = {g + "/" + k: rng.standard_normal(s).astype(np.float32) for g in ("theta", "adam_m", "adam_v")
            for k, s in old.shapes().items()}
    path = str(tmp_path / "c.c2v_b200")
    prefix, entries, _ = checkpoint_header(vars(old), 7, 0, True)
    write_checkpoint(path, prefix, [full[e["name"]] for e in entries])
    sentinel = np.float32(-12345.5)
    straddled = 0
    for r in range(world):
        y0, y1 = target_row_block(Y_new, r, world)
        straddled += y0 < Y_old < y1
        per = {"tok": -(-T_new // world), "path": -(-P_new // world)}
        out = {}
        for g in ("theta", "adam_m", "adam_v"):
            out[g + "/tok"] = np.full((per["tok"], d), sentinel, np.float32)
            out[g + "/path"] = np.full((per["path"], d), sentinel, np.float32)
            out[g + "/tgt"] = np.full((y1 - y0, D), sentinel, np.float32)
            out[g + "/W"] = np.full((3 * d, D), sentinel, np.float32)
            out[g + "/a"] = np.full((D,), sentinel, np.float32)
        meta = read_checkpoint_part(path, r, world, (y0, y1), out)
        assert meta["adam_t"] == 7
        for g in ("theta", "adam_m", "adam_v"):
            for name, n_old in (("tok", T_old), ("path", P_old)):
                got = out[g + "/" + name]
                for i in range(got.shape[0]):
                    row = i * world + r                           # local row i holds global row i * W + r
                    if row < n_old:
                        assert np.array_equal(got[i], full[g + "/" + name][row]), (g, name, r, i)
                    else:
                        assert np.all(got[i] == sentinel), (g, name, r, i)
            got = out[g + "/tgt"]
            for i in range(got.shape[0]):
                row = y0 + i
                if row < Y_old:
                    assert np.array_equal(got[i], full[g + "/tgt"][row]), (g, r, i)
                else:
                    assert np.all(got[i] == sentinel), (g, r, i)
            assert np.array_equal(out[g + "/W"], full[g + "/W"]) and np.array_equal(out[g + "/a"], full[g + "/a"])
    assert world == 1 or straddled == 1
