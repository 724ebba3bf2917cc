"""Run configuration with the reference's surface (reference config.py:9-277), TensorFlow-free.

Same attribute names, flags, derived properties and `verify()` errors as the reference's Config so
that code written against it (the model base class, the reader, the vocabularies) runs unchanged;
the one addition is two more values of `--framework`: ``b200`` (the CUDA path-attention engine with
the TensorFlow backend's numerics; the default here) and ``b200-keras`` (the same engine with the
Keras backend's initialisers, optimizer epsilon, scores and evaluation schedule).
"""
from __future__ import annotations

import logging
import math
import os
import sys
from argparse import ArgumentParser
from typing import Iterator, Optional, Tuple

FRAMEWORKS = ("b200", "b200-keras", "tensorflow", "keras")

# name -> default, in the groups the reference uses (config.py:46-70)
_TRAINING_DEFAULTS = {
    "NUM_TRAIN_EPOCHS": 20,
    "SAVE_EVERY_EPOCHS": 1,
    "TRAIN_BATCH_SIZE": 1024,
    "TEST_BATCH_SIZE": 1024,
    "TOP_K_WORDS_CONSIDERED_DURING_PREDICTION": 10,
    "NUM_BATCHES_TO_LOG_PROGRESS": 100,
    "NUM_TRAIN_BATCHES_TO_EVALUATE": 1800,
    "READER_NUM_PARALLEL_BATCHES": 6,
    "SHUFFLE_BUFFER_SIZE": 10000,
    "CSV_BUFFER_SIZE": 100 * 1024 * 1024,
    "MAX_TO_KEEP": 10,
}
_MODEL_DEFAULTS = {
    "MAX_CONTEXTS": 200,
    "MAX_TOKEN_VOCAB_SIZE": 1301136,
    "MAX_TARGET_VOCAB_SIZE": 261245,
    "MAX_PATH_VOCAB_SIZE": 911417,
    "DEFAULT_EMBEDDINGS_SIZE": 128,
    "DROPOUT_KEEP_RATE": 0.75,
    "SEPARATE_OOV_AND_PAD": False,
}
_ARG_FIELDS = {   # attribute -> (argparse dest, default when absent)
    "PREDICT": ("predict", False),
    "MODEL_SAVE_PATH": ("save_path", None),
    "MODEL_LOAD_PATH": ("load_path", None),
    "TRAIN_DATA_PATH_PREFIX": ("data_path", None),
    "TEST_DATA_PATH": ("test_path", ""),
    "RELEASE": ("release", False),
    "EXPORT_CODE_VECTORS": ("export_code_vectors", False),
    "SAVE_W2V": ("save_w2v", None),
    "SAVE_T2V": ("save_t2v", None),
    "VERBOSE_MODE": ("verbose_mode", 0),
    "LOGS_PATH": ("logs_path", None),
    "USE_TENSORBOARD": ("use_tensorboard", False),
}


def _is_set(option: str) -> property:
    """True when a path-like option was given (config.py:147-161)."""
    return property(lambda self: bool(getattr(self, option)))


def _batches_of(examples: str, batch: str) -> property:
    """ceil(examples / batch), 0 while the batch size is unset (config.py:163-169)."""
    return property(lambda self: math.ceil(getattr(self, examples) / getattr(self, batch)) if getattr(self, batch) else 0)


def _only_if(flag: str, value) -> property:
    """A derived path that exists only in the mode `flag` names, else None (config.py:177-230)."""
    return property(lambda self: value(self) if getattr(self, flag) else None)


class Config:
    @classmethod
    def arguments_parser(cls) -> ArgumentParser:
        """The reference's command line (config.py:11-44) plus `--framework b200`."""
        p = ArgumentParser()
        p.add_argument("-d", "--data", dest="data_path", required=False, help="path to preprocessed dataset")
        p.add_argument("-te", "--test", dest="test_path", metavar="FILE", required=False, default="",
                       help="path to test file")
        p.add_argument("-s", "--save", dest="save_path", metavar="FILE", required=False,
                       help="path to save the model file")
        p.add_argument("-w2v", "--save_word2v", "--save_w2v", dest="save_w2v", metavar="FILE", required=False,
                       help="save token vectors in word2vec text format")
        p.add_argument("-t2v", "--save_target2v", "--save_t2v", dest="save_t2v", metavar="FILE", required=False,
                       help="save target vectors in word2vec text format")
        p.add_argument("-l", "--load", dest="load_path", metavar="FILE", required=False,
                       help="path to load the model from")
        p.add_argument("--export_code_vectors", action="store_true", required=False,
                       help="export code vectors for the given examples")
        p.add_argument("--release", action="store_true",
                       help="when loading a trained model, re-save it without optimizer state")
        p.add_argument("--predict", action="store_true", help="execute the interactive prediction shell")
        p.add_argument("-fw", "--framework", dest="dl_framework", choices=list(FRAMEWORKS), default="b200",
                       help="model backend to use")
        p.add_argument("-v", "--verbose", dest="verbose_mode", type=int, required=False, default=1,
                       help="verbose mode (should be in {0,1,2})")
        p.add_argument("-lp", "--logs-path", dest="logs_path", metavar="FILE", required=False,
                       help="path to store logs into; if not given logs are not saved to file")
        p.add_argument("-tb", "--tensorboard", dest="use_tensorboard", action="store_true",
                       help="accepted for compatibility; ignored by the b200 backend")
        return p

    def __init__(self, set_defaults: bool = False, load_from_args: bool = False, verify: bool = False):
        for name in _TRAINING_DEFAULTS:
            setattr(self, name, 0)
        for name, default in _MODEL_DEFAULTS.items():
            setattr(self, name, type(default)())
        self.TOKEN_EMBEDDINGS_SIZE = 0
        self.PATH_EMBEDDINGS_SIZE = 0
        self.CODE_VECTOR_SIZE = 0
        self.TARGET_EMBEDDINGS_SIZE = 0
        for name, (_, default) in _ARG_FIELDS.items():
            setattr(self, name, default)
        self.DL_FRAMEWORK = ""
        # filled by Code2VecModelBase._init_num_of_examples()
        self.NUM_TRAIN_EXAMPLES = 0
        self.NUM_TEST_EXAMPLES = 0
        self.__logger: Optional[logging.Logger] = None
        self.__quiet = False
        if set_defaults:
            self.set_defaults()
        if load_from_args:
            self.load_from_args()
        if verify:
            self.verify()

    def set_defaults(self):
        for name, value in _TRAINING_DEFAULTS.items():
            setattr(self, name, value)
        for name, value in _MODEL_DEFAULTS.items():
            setattr(self, name, value)
        self.TOKEN_EMBEDDINGS_SIZE = self.DEFAULT_EMBEDDINGS_SIZE
        self.PATH_EMBEDDINGS_SIZE = self.DEFAULT_EMBEDDINGS_SIZE
        self.CODE_VECTOR_SIZE = self.context_vector_size
        self.TARGET_EMBEDDINGS_SIZE = self.CODE_VECTOR_SIZE

    def load_from_args(self, argv=None):
        args = self.arguments_parser().parse_args(argv)
        for name, (dest, _) in _ARG_FIELDS.items():
            setattr(self, name, getattr(args, dest))
        self.DL_FRAMEWORK = args.dl_framework or "b200"

    # ---- derived values (config.py:143-230): declared through the three helpers below the class ----
    context_vector_size = property(
        lambda self: 2 * self.TOKEN_EMBEDDINGS_SIZE + self.PATH_EMBEDDINGS_SIZE,
        doc="width of one context: source-token, path and target-token embeddings side by side")

    is_training = _is_set("TRAIN_DATA_PATH_PREFIX")
    is_loading = _is_set("MODEL_LOAD_PATH")
    is_saving = _is_set("MODEL_SAVE_PATH")
    is_testing = _is_set("TEST_DATA_PATH")

    train_steps_per_epoch = _batches_of("NUM_TRAIN_EXAMPLES", "TRAIN_BATCH_SIZE")
    test_steps = _batches_of("NUM_TEST_EXAMPLES", "TEST_BATCH_SIZE")

    train_data_path = _only_if("is_training", lambda self: self.TRAIN_DATA_PATH_PREFIX + ".train.c2v")
    word_freq_dict_path = _only_if("is_training", lambda self: self.TRAIN_DATA_PATH_PREFIX + ".dict.c2v")
    entire_model_load_path = _only_if("is_loading", lambda self: self.get_entire_model_path(self.MODEL_LOAD_PATH))
    model_weights_load_path = _only_if("is_loading", lambda self: self.get_model_weights_path(self.MODEL_LOAD_PATH))
    entire_model_save_path = _only_if("is_saving", lambda self: self.get_entire_model_path(self.MODEL_SAVE_PATH))
    model_weights_save_path = _only_if("is_saving", lambda self: self.get_model_weights_path(self.MODEL_SAVE_PATH))
    model_load_dir = property(lambda self: self.MODEL_LOAD_PATH.rpartition("/")[0])

    def data_path(self, is_evaluating: bool = False):
        return self.TEST_DATA_PATH if is_evaluating else self.train_data_path

    def batch_size(self, is_evaluating: bool = False):
        return self.TEST_BATCH_SIZE if is_evaluating else self.TRAIN_BATCH_SIZE

    @staticmethod
    def get_vocabularies_path_from_model_path(model_file_path: str) -> str:
        """`dictionaries.bin` lives beside the model files."""
        folder, slash, _ = model_file_path.rpartition("/")
        return folder + slash + "dictionaries.bin"

    @staticmethod
    def get_entire_model_path(model_path: str) -> str:
        return model_path + "__entire-model"

    @staticmethod
    def get_model_weights_path(model_path: str) -> str:
        return model_path + "__only-weights"

    def verify(self):
        """Same failure conditions and messages as the reference (config.py:232-239)."""
        if not self.is_training and not self.is_loading:
            raise ValueError("Must train or load a model.")
        if self.is_loading and not os.path.isdir(self.model_load_dir):
            raise ValueError("Model load dir `{model_load_dir}` does not exist.".format(
                model_load_dir=self.model_load_dir))
        if self.DL_FRAMEWORK not in set(FRAMEWORKS):
            raise ValueError("config.DL_FRAMEWORK must be in {'b200', 'b200-keras', 'tensorflow', 'keras'}.")

    def __iter__(self) -> Iterator[Tuple[str, object]]:
        """(name, value) of every non-callable public attribute -- the start-up config dump."""
        for name in dir(self):
            if name.startswith("__") or name.startswith("_Config__"):
                continue
            try:
                value = getattr(self, name, None)
            except Exception:
                value = None
            if callable(value):
                continue
            yield name, value

    # ---- logging (config.py:253-277) ---------------------------------------------------------
    def get_logger(self) -> logging.Logger:
        if self.__logger is None:
            logger = logging.getLogger("code2vec")
            logger.setLevel(logging.INFO)
            logger.handlers = []
            logger.propagate = 0
            fmt = logging.Formatter("%(asctime)s %(levelname)-8s %(message)s")
            sinks = []
            if self.VERBOSE_MODE >= 1:
                sinks.append(logging.StreamHandler(sys.stdout))
            if self.LOGS_PATH:
                sinks.append(logging.FileHandler(self.LOGS_PATH))
            for h in sinks:
                h.setLevel(logging.INFO)
                h.setFormatter(fmt)
                logger.addHandler(h)
            self.__logger = logger
        return self.__logger

    def log(self, msg):
        if not self.__quiet:
            self.get_logger().info(msg)

    def quiet(self):
        """Drop every later log() line: the ranks other than 0 of a multi-GPU run, where rank 0 logs for all."""
        self.__quiet = True
