"""The model-backend seam of the reference (model_base.py:11-182), restated for the engine's backends.

A backend written against the reference's `Code2VecModelBase` finds the same names here: the two
result tuples, the constructor's order of events (verify the configuration, size the datasets,
build or load the vocabularies, create or load the inner model, initialise), the helpers every
backend shares (checkpoint directory + vocabulary saving, word2vec export, code-vector lines, the
attention dictionary of a prediction) and the six methods a backend must provide.  What the helpers
print and write is pinned against the real module (tests/test_host_surface2.py).
"""
from __future__ import annotations

import abc
import os
from typing import Dict, Iterable, List, NamedTuple, Optional, Tuple

import numpy as np

from .common import common
from .config import Config
from .vocabularies import Code2VecVocabs, VocabType

_RULE_WIDTH = 69                                   # width of the start-up banner (model_base.py:52-60)


def _rule(title: str = "") -> str:
    """A banner line: dashes, optionally around a centred title (odd leftovers go to the right)."""
    if not title:
        return "-" * _RULE_WIDTH
    body = " %s " % title
    left = (_RULE_WIDTH - len(body)) // 2
    return "-" * left + body + "-" * (_RULE_WIDTH - len(body) - left)


def _cached_line_count(dataset_path: str) -> int:
    """Number of examples of a `.c2v` file, remembered next to it in `<file>.num_examples`
    (model_base.py:86-96): an existing side-car wins over the file itself."""
    note = dataset_path + ".num_examples"
    try:
        with open(note, "r") as fh:
            return int(fh.readline())
    except FileNotFoundError:
        count = common.count_lines_in_file(dataset_path)
        with open(note, "w") as fh:
            fh.write(str(count))
        return count


class ModelEvaluationResults(NamedTuple):
    """What `evaluate()` returns (model_base.py:11-26).  `loss` is only filled by the Keras-numerics backend."""
    topk_acc: float
    subtoken_precision: float
    subtoken_recall: float
    subtoken_f1: float
    loss: Optional[float] = None

    def __str__(self):
        shown = [("topk_acc", self.topk_acc), ("precision", self.subtoken_precision), ("recall", self.subtoken_recall),
                 ("F1", self.subtoken_f1)]
        if self.loss is not None:
            shown.insert(0, ("loss", self.loss))
        return ", ".join("%s: %s" % pair for pair in shown)


class ModelPredictionResults(NamedTuple):
    """One predicted method (model_base.py:29-34)."""
    original_name: str
    topk_predicted_words: np.ndarray
    topk_predicted_words_scores: np.ndarray
    attention_per_context: Dict[Tuple[str, str, str], float]
    code_vector: Optional[np.ndarray] = None


class Code2VecModelBase(abc.ABC):
    # ---- construction: the reference's order of events (model_base.py:38-50) ---------------------
    def __init__(self, config: Config):
        self.config = config
        config.verify()
        self._log_creating_model()
        if not config.RELEASE:                      # a release run has no datasets to size
            self._init_num_of_examples()
        self._log_model_configuration()
        self.vocabs = self._make_vocabs()
        self.vocabs.target_vocab.get_index_to_word_lookup_table()
        self._load_or_create_inner_model()
        self._initialize()

    def load_or_build(self):
        self.vocabs = self._make_vocabs()
        self._load_or_create_inner_model()

    def _make_vocabs(self) -> Code2VecVocabs:
        return Code2VecVocabs(self.config)

    def _load_or_create_inner_model(self):
        (self._load_inner_model if self.config.is_loading else self._create_inner_model)()

    # ---- the backend's part ----------------------------------------------------------------------
    @abc.abstractmethod
    def train(self):
        """Run the training loop over `config.train_data_path` (saving / evaluating on the backend's schedule)."""

    @abc.abstractmethod
    def evaluate(self) -> Optional[ModelEvaluationResults]:
        """Score `config.TEST_DATA_PATH`; None when the run only releases a model."""

    @abc.abstractmethod
    def predict(self, predict_data_lines: Iterable[str]) -> List[ModelPredictionResults]:
        """One result per input line (a line = the extractor's output for one method)."""

    @abc.abstractmethod
    def _save_inner_model(self, path):
        """Write the backend's own checkpoint for the model path `path`."""

    @abc.abstractmethod
    def _load_inner_model(self):
        """Restore the backend from `config.MODEL_LOAD_PATH`."""

    @abc.abstractmethod
    def _get_vocab_embedding_as_np_array(self, vocab_type: VocabType) -> np.ndarray:
        """The `[vocabulary size, dimension]` embedding matrix of one vocabulary."""

    def _create_inner_model(self):                  # optional hooks (model_base.py:161-170)
        pass

    def _initialize(self):
        pass

    def close_session(self):
        pass

    # ---- logging -----------------------------------------------------------------------------------
    @property
    def logger(self):
        return self.config.get_logger()

    def log(self, msg):
        self.logger.info(msg)

    def _log_creating_model(self):
        for line in ["", ""] + [_rule()] * 2 + [_rule("Creating code2vec model")] + [_rule()] * 2:
            self.log(line)

    def _log_model_configuration(self):
        settings = list(self.config)
        column = 2 + max(len(name) for name, _ in settings)
        self.log(_rule())
        self.log(_rule("Configuration - Hyper Parameters"))
        for name, value in settings:
            self.log(name.ljust(column) + str(value))
        self.log(_rule())

    # ---- dataset sizes -------------------------------------------------------------------------------
    _get_num_of_examples_for_dataset = staticmethod(_cached_line_count)

    def _init_num_of_examples(self):
        cfg = self.config
        self.log("Checking number of examples ...")
        for wanted, attr, path, label in ((cfg.is_training, "NUM_TRAIN_EXAMPLES", lambda: cfg.train_data_path, "train"),
                                          (cfg.is_testing, "NUM_TEST_EXAMPLES", lambda: cfg.TEST_DATA_PATH, "test")):
            if wanted:
                setattr(cfg, attr, self._get_num_of_examples_for_dataset(path()))
                self.log("    Number of %s examples: %s" % (label, getattr(cfg, attr)))

    # ---- what every backend shares ---------------------------------------------------------------------
    def save(self, model_save_path=None):
        """Vocabularies (`dictionaries.bin` beside the model) + the backend's checkpoint (model_base.py:102-109)."""
        target = model_save_path if model_save_path is not None else self.config.MODEL_SAVE_PATH
        folder = target.rpartition("/")[0]
        if folder:
            os.makedirs(folder, exist_ok=True)
        self.vocabs.save(self.config.get_vocabularies_path_from_model_path(target))
        self._save_inner_model(target)

    def save_word2vec_format(self, dest_save_path: str, vocab_type: VocabType):
        if vocab_type not in VocabType:
            raise ValueError("`vocab_type` should be `VocabType.Token`, `VocabType.Target` or `VocabType.Path`.")
        vocab = self.vocabs.get(vocab_type)
        with open(dest_save_path, "w") as out:
            common.save_word2vec_file(out, vocab.index_to_word, self._get_vocab_embedding_as_np_array(vocab_type))

    def _write_code_vectors(self, file, code_vectors):
        """One space-joined vector per line: the `<test file>.vectors` format (model_base.py:111-113)."""
        file.writelines(" ".join(str(x) for x in vector) + "\n" for vector in code_vectors)

    def _get_attention_weight_per_context(self, path_source_strings: Iterable[str], path_strings: Iterable[str],
                                          path_target_strings: Iterable[str],
                                          attention_weights: Iterable[float]) -> Dict[Tuple[str, str, str], float]:
        """{(source token, path, target token): attention}.  Keyed by strings, so a context that occurs more
        than once in the bag keeps the weight of its LAST occurrence (model_base.py:115-129)."""
        weights = np.asarray(attention_weights)
        weights = weights.reshape(weights.shape[0]) if weights.ndim == 2 else weights
        text = common.binary_to_string
        triples = zip(map(text, path_source_strings), map(text, path_strings), map(text, path_target_strings))
        return dict(zip(triples, weights))
