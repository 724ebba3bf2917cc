"""Vocabularies with the reference's surface and on-disk formats (reference vocabularies.py),
TensorFlow-free: the tf.lookup.StaticHashTable lookups (vocabularies.py:108-139) become plain
dict lookups on the host -- string<->index translation never touches the GPU path.

Kept verbatim in meaning: special words come first (index 0; :51-55), three special-word modes
(:22-35,204-209), frequency-sorted truncation to MAX_*_VOCAB_SIZE (:99-106), the pickle layout of
``dictionaries.bin`` (token, target, path; three pickles each, specials excluded; :57-66,211-218)
and of ``<data>.dict.c2v`` (:220-230), and the load-time consistency error (:78-89).
"""
from __future__ import annotations

import os
import pickle
from argparse import Namespace
from enum import Enum
from typing import Dict, Iterable, NamedTuple, Optional, Set

import numpy as np

from .common import common
from .config import Config


class VocabType(Enum):
    Token = 1
    Target = 2
    Path = 3


SpecialVocabWordsType = Namespace

_SpecialVocabWords_OnlyOov = Namespace(OOV="<OOV>")
_SpecialVocabWords_SeparateOovPad = Namespace(PAD="<PAD>", OOV="<OOV>")
_SpecialVocabWords_JoinedOovPad = Namespace(PAD_OR_OOV="<PAD_OR_OOV>", PAD="<PAD_OR_OOV>", OOV="<PAD_OR_OOV>")


def _unique_specials(special_words: SpecialVocabWordsType) -> list:
    return common.get_unique_list(vars(special_words).values())


class Vocab:
    def __init__(self, vocab_type: VocabType, words: Iterable[str], special_words: Optional[SpecialVocabWordsType] = None):
        self.vocab_type = vocab_type
        self.special_words: SpecialVocabWordsType = special_words if special_words is not None else Namespace()
        self.word_to_index: Dict[str, int] = {}
        self.index_to_word: Dict[int, str] = {}
        for word in list(_unique_specials(self.special_words)) + list(words):
            idx = len(self.index_to_word)     # positions count duplicates too, as enumerate() does in the reference
            self.word_to_index[word] = idx
            self.index_to_word[idx] = word
        self.size = len(self.word_to_index)
        self._index_array_cache = None

    # ---- persistence: specials are not stored (historical format) ----------------------------
    def save_to_file(self, file):
        n_special = len(_unique_specials(self.special_words))
        pickle.dump({w: i for w, i in self.word_to_index.items() if i >= n_special}, file)
        pickle.dump({i: w for i, w in self.index_to_word.items() if i >= n_special}, file)
        pickle.dump(self.size - n_special, file)

    @classmethod
    def load_from_file(cls, vocab_type: VocabType, file, special_words: SpecialVocabWordsType) -> "Vocab":
        specials = _unique_specials(special_words)
        word_to_index_wo = pickle.load(file)
        index_to_word_wo = pickle.load(file)
        size_wo = pickle.load(file)
        assert len(index_to_word_wo) == len(word_to_index_wo) == size_wo
        lowest = min(index_to_word_wo.keys())
        if lowest != len(specials):
            raise ValueError(
                "Error while attempting to load vocabulary `{vocab_type}` from file `{file_path}`. "
                "The stored vocabulary has minimum word index {min_word_idx}, "
                "while expecting minimum word index to be {nr_special_words} "
                "because having to use {nr_special_words} special words, which are: {special_words}. "
                "Please check the parameter `config.SEPARATE_OOV_AND_PAD`.".format(
                    vocab_type=vocab_type, file_path=getattr(file, "name", "?"), min_word_idx=lowest,
                    nr_special_words=len(specials), special_words=special_words))
        vocab = cls(vocab_type, [], special_words)
        vocab.word_to_index = dict(word_to_index_wo)
        vocab.index_to_word = dict(index_to_word_wo)
        for i, w in enumerate(specials):
            vocab.word_to_index[w] = i
            vocab.index_to_word[i] = w
        vocab.size = size_wo + len(specials)
        return vocab

    @classmethod
    def create_from_freq_dict(cls, vocab_type: VocabType, word_to_count: Dict[str, int], max_size: int,
                              special_words: Optional[SpecialVocabWordsType] = None):
        by_count_desc = sorted(word_to_count, key=word_to_count.get, reverse=True)   # stable: ties keep dict order
        return cls(vocab_type, by_count_desc[:max_size], special_words)

    # ---- lookups (host-side replacements for the StaticHashTables) ----------------------------
    def get_word_to_index_lookup_table(self):
        return self.word_to_index

    def get_index_to_word_lookup_table(self):
        return self.index_to_word

    def lookup_index(self, words) -> np.ndarray:
        """word(s) -> int32 index, unknown words -> OOV index (vocabularies.py:123-127,135-136)."""
        oov = self.word_to_index[self.special_words.OOV]
        get = self.word_to_index.get
        if isinstance(words, str):
            return np.int32(get(words, oov))
        return np.fromiter((get(w, oov) for w in words), dtype=np.int32, count=len(words))

    def lookup_word(self, indices):
        """index/indices -> word(s), unknown indices -> OOV word (vocabularies.py:129-133,138-139)."""
        oov = self.special_words.OOV
        get = self.index_to_word.get
        if np.isscalar(indices):
            return get(int(indices), oov)
        arr = np.asarray(indices)
        flat = [get(int(i), oov) for i in arr.reshape(-1)]
        return np.array(flat, dtype=object).reshape(arr.shape)


WordFreqDictType = Dict[str, int]


def extend_vocab(loaded: Vocab, word_to_count: Dict[str, int], max_size: int) -> Vocab:
    """`loaded` with the words a model trained from scratch on `word_to_count` would hold appended (C2V_EXTEND_VOCAB=1,
    DESIGN.md §6m): every loaded word, the special words included, keeps its index, and each word of
    create_from_freq_dict(word_to_count, max_size) that `loaded` does not hold follows, in that function's order.  Old
    rows never move, so a table grown to the merged size keeps the loaded table as its leading rows."""
    fresh = Vocab.create_from_freq_dict(loaded.vocab_type, word_to_count, max_size, loaded.special_words)
    merged = Vocab(loaded.vocab_type, [], loaded.special_words)
    merged.word_to_index = dict(loaded.word_to_index)
    merged.index_to_word = dict(loaded.index_to_word)
    merged.size = loaded.size
    for i in range(len(fresh.index_to_word)):
        word = fresh.index_to_word[i]
        if word not in merged.word_to_index:
            merged.word_to_index[word] = merged.size
            merged.index_to_word[merged.size] = word
            merged.size += 1
    return merged


class Code2VecWordFreqDicts(NamedTuple):
    """The three histograms of `<data>.dict.c2v`, in the order the file stores them (preprocess.py:12-20)."""
    token_to_count: WordFreqDictType
    path_to_count: WordFreqDictType
    target_to_count: WordFreqDictType


class _Slot(NamedTuple):
    """How one of the three vocabularies is wired: attribute on Code2VecVocabs, histogram field, size limit, log name."""
    kind: VocabType
    attr: str
    histogram: str
    limit: str
    label: str


_SLOTS = {
    VocabType.Token: _Slot(VocabType.Token, "token_vocab", "token_to_count", "MAX_TOKEN_VOCAB_SIZE", "token"),
    VocabType.Path: _Slot(VocabType.Path, "path_vocab", "path_to_count", "MAX_PATH_VOCAB_SIZE", "path"),
    VocabType.Target: _Slot(VocabType.Target, "target_vocab", "target_to_count", "MAX_TARGET_VOCAB_SIZE", "target"),
}
_BUILD_ORDER = (VocabType.Token, VocabType.Path, VocabType.Target)      # creation and its log lines (vocabularies.py:188-202)
_DISK_ORDER = (VocabType.Token, VocabType.Target, VocabType.Path)       # dictionaries.bin (vocabularies.py:211-218)


class Code2VecVocabs:
    """The token / path / target vocabularies of a model: built from the training histograms, or read
    back from the `dictionaries.bin` stored next to a saved model (reference vocabularies.py:142-243).

    extend: a run that loads and trains extends the loaded vocabularies by the training histograms' words (extend_vocab);
    loaded_sizes then holds each vocabulary's size before the extension, else it is None."""

    def __init__(self, config: Config, extend: bool = False):
        self.config = config
        self.token_vocab: Optional[Vocab] = None
        self.path_vocab: Optional[Vocab] = None
        self.target_vocab: Optional[Vocab] = None
        self.loaded_sizes: Optional[Dict[VocabType, int]] = None
        self._already_saved_in_paths: Set[str] = set()
        self._load_or_create(extend)

    # ---- which special words a vocabulary starts with (vocabularies.py:204-209) -----------------
    def _get_special_words_by_vocab_type(self, vocab_type: VocabType) -> SpecialVocabWordsType:
        if self.config.SEPARATE_OOV_AND_PAD:
            return _SpecialVocabWords_OnlyOov if vocab_type is VocabType.Target else _SpecialVocabWords_SeparateOovPad
        return _SpecialVocabWords_JoinedOovPad

    # ---- construction --------------------------------------------------------------------------------
    def _load_or_create(self, extend: bool = False):
        cfg = self.config
        assert cfg.is_training or cfg.is_loading
        if not cfg.is_loading:
            self._create_from_word_freq_dict()
            return
        stored = cfg.get_vocabularies_path_from_model_path(cfg.MODEL_LOAD_PATH)
        if not os.path.isfile(stored):
            raise ValueError("Model dictionaries file is not found in model load dir. "
                             "Expecting file `{vocabularies_load_path}`.".format(vocabularies_load_path=stored))
        self._load_from_path(stored)
        if extend and cfg.is_training:
            self._extend_from_word_freq_dict()
            self._already_saved_in_paths.discard(stored)                # the file holds the loaded vocabularies only

    def _load_from_path(self, vocabularies_load_path: str):
        assert os.path.exists(vocabularies_load_path)
        self.config.log("Loading model vocabularies from: `%s` ... " % vocabularies_load_path)
        with open(vocabularies_load_path, "rb") as fh:
            for kind in _DISK_ORDER:
                setattr(self, _SLOTS[kind].attr, Vocab.load_from_file(kind, fh, self._get_special_words_by_vocab_type(kind)))
        self.config.log("Done loading model vocabularies.")
        self._already_saved_in_paths.add(vocabularies_load_path)        # no need to write the same file back

    def _load_word_freq_dict(self) -> Code2VecWordFreqDicts:
        cfg = self.config
        assert cfg.is_training
        cfg.log("Loading word frequencies dictionaries from: %s ... " % cfg.word_freq_dict_path)
        with open(cfg.word_freq_dict_path, "rb") as fh:                  # a fourth pickle (the example count) follows
            histograms = Code2VecWordFreqDicts(*(pickle.load(fh) for _ in Code2VecWordFreqDicts._fields))
        cfg.log("Done loading word frequencies dictionaries.")
        return histograms

    def _create_from_word_freq_dict(self):
        histograms = self._load_word_freq_dict()
        self.config.log("Word frequencies dictionaries loaded. Now creating vocabularies.")
        for kind in _BUILD_ORDER:
            slot = _SLOTS[kind]
            vocab = Vocab.create_from_freq_dict(kind, getattr(histograms, slot.histogram), getattr(self.config, slot.limit),
                                                special_words=self._get_special_words_by_vocab_type(kind))
            setattr(self, slot.attr, vocab)
            self.config.log("Created %s vocab. size: %d" % (slot.label, vocab.size))

    def _extend_from_word_freq_dict(self):
        histograms = self._load_word_freq_dict()
        self.loaded_sizes = {}
        for kind in _BUILD_ORDER:
            slot = _SLOTS[kind]
            loaded = getattr(self, slot.attr)
            merged = extend_vocab(loaded, getattr(histograms, slot.histogram), getattr(self.config, slot.limit))
            setattr(self, slot.attr, merged)
            self.loaded_sizes[kind] = loaded.size
            self.config.log("Extended %s vocab (C2V_EXTEND_VOCAB=1): %d + %d new words = %d" % (
                slot.label, loaded.size, merged.size - loaded.size, merged.size))

    # ---- use -----------------------------------------------------------------------------------------
    def get(self, vocab_type: VocabType) -> Vocab:
        if not isinstance(vocab_type, VocabType):
            raise ValueError("`vocab_type` should be `VocabType.Token`, `VocabType.Target` or `VocabType.Path`.")
        return getattr(self, _SLOTS[vocab_type].attr)

    def save(self, vocabularies_save_path: str):
        """Writes `dictionaries.bin` once per destination (vocabularies.py:211-218)."""
        if vocabularies_save_path in self._already_saved_in_paths:
            return
        with open(vocabularies_save_path, "wb") as fh:
            for kind in _DISK_ORDER:
                self.get(kind).save_to_file(fh)
        self._already_saved_in_paths.add(vocabularies_save_path)
